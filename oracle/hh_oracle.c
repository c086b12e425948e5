/* oracle/hh_oracle.c -- TEST INFRASTRUCTURE (the parity oracle), NOT product code.
 *
 * A scalar, per-target CPU restatement of the reference's hot path, written from the behaviour
 * documented in SURVEY.md App. A and checked bit-for-bit against the compiled reference
 * (oracle/_ref/libhhref_shim.so, AVX2 / no-FMA build = the official release flags) by
 * tests/test_oracle_vs_ref.py and against the committed fixtures in tests/golden/.
 * PARITY PINNED: yes (reference run in this container; goldens committed with their generator
 * tests/golden/make_golden.py).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load this library.
 * The product (hh-suite_b200/csrc) never links or calls it.
 *
 * Build: gcc -O2 -ffp-contract=off -fno-fast-math -fPIC -shared  (no -mfma: every mul/add is a
 * separately rounded IEEE fp32 operation, as in the reference's -mavx2 build).
 *
 * Data layout (shared with include/hhg.h):
 *   p  : float[(L+2)*20]   p[i*20+a], columns 0..L+1 (reference HMM::p, src/hhhmm.h:153)
 *   tr : float[(L+1)*7]    tr[i*7+k], k in the reference enum order M2M,M2I,M2D,I2M,I2I,D2M,D2D
 *                          (src/hhdecl.h:68), log2 transition probabilities
 *   ss : u8[L+2]           ss[i] = ss_pred[i]*MAXCF + ss_conf[i]  (src/hhhmmsimd.cpp:133), MAXCF=11
 *   S33: float[44*44]      S33[q_ss*44 + t_ss]   (src/hhdecl.h:53-55: NSSPRED=4, MAXCF=11)
 *   bt : u8[(Lq+1)*(Lt+1)] bt[i*(Lt+1)+j], bit layout of ViterbiMatrix (src/hhviterbimatrix-inl.h)
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

enum { M2M = 0, M2I = 1, M2D = 2, I2M = 3, I2I = 4, D2M = 5, D2D = 6 };
enum { ST_STOP = 0, ST_MM = 2, ST_GD = 3, ST_IM = 4, ST_DG = 5, ST_MI = 6 };

static inline uint32_t f2u(float x) { uint32_t u; memcpy(&u, &x, 4); return u; }
static inline float u2f(uint32_t u) { float x; memcpy(&x, &u, 4); return x; }

/* Follows Viterbi::ScalarProd20Vec, src/hhviterbi.h:126-190: four partial sums over a = k mod 4,
 * accumulated in increasing a, combined as (r0+r1)+(r2+r3). */
static inline float dot20(const float* q, const float* t) {
  float r0 = t[0] * q[0], r1 = t[1] * q[1], r2 = t[2] * q[2], r3 = t[3] * q[3];
  for (int m = 1; m < 5; ++m) {
    r0 = t[4 * m + 0] * q[4 * m + 0] + r0;
    r1 = t[4 * m + 1] * q[4 * m + 1] + r1;
    r2 = t[4 * m + 2] * q[4 * m + 2] + r2;
    r3 = t[4 * m + 3] * q[4 * m + 3] + r3;
  }
  r0 = r0 + r1;
  r2 = r2 + r3;
  return r0 + r2;
}

/* Follows log2f4, src/hhutil-inl.h:509-541 (LOG_POLY_DEGREE 4 => POLY3). */
static inline float log2f4_scalar(float x) {
  uint32_t i = f2u(x);
  float e = (float)((int32_t)((i & 0x7F800000u) >> 23) - 127);
  float m = u2f((i & 0x007FFFFFu) | 0x3F800000u);
  float p = -0.107254423828329604454f;
  p = p * m + 0.688243882994381274313f;
  p = p * m + -1.75647175389045657003f;
  p = p * m + 2.61761038894603480148f;
  p = p * (m - 1.0f);
  return p + e;
}

/* The forward pass. Follows Viterbi::AlignWith[Out]CellOff[AndSS],
 * src/hhviterbialgorithm.cpp:77-497 (one lane of the SIMD batch, no padding columns).
 *   q_ss/t_ss/S33 : all non-NULL selects the *AndSS variants (PRED_PRED mode, :199-211,279)
 *   celloff       : non-NULL selects the *CellOff variants (:373-392); bytes != 0 are off
 * Returns 0. Outputs: *score,*i2,*j2 (ViterbiResult, src/hhviterbi.h:21), bt bytes (bits 0-6). */
int hho_viterbi_align(int Lq, const float* q_p, const float* q_tr, const uint8_t* q_ss,
                      int Lt, const float* t_p, const float* t_tr, const uint8_t* t_ss,
                      const float* S33, float ssw, const uint8_t* celloff, int local, float egq,
                      float egt, float shift, float* score, int* i2, int* j2, uint8_t* bt) {
  const float smin = local ? 0.0f : -FLT_MAX;
  const int use_ss = (q_ss && t_ss && S33);
  float* sMM = (float*)malloc(sizeof(float) * 5 * (size_t)(Lt + 1));
  float *sDG = sMM + (Lt + 1), *sMI = sDG + (Lt + 1), *sGD = sMI + (Lt + 1), *sIM = sGD + (Lt + 1);
  float best = -FLT_MAX;
  int bi = 0, bj = 0;
  for (int j = 0; j <= Lt; ++j) {           /* :145-153 */
    sMM[j] = (float)(-j) * egt;
    sDG[j] = sMI[j] = sGD[j] = sIM[j] = -FLT_MAX;
  }
  for (int i = 1; i <= Lq; ++i) {
    float dMM = (float)(-(i - 1)) * egq;      /* :161-165 */
    float dIM = -FLT_MAX, dMI = -FLT_MAX, dDG = -FLT_MAX, dGD = -FLT_MAX;
    sMM[0] = (float)(-i) * egq;               /* :169-173 */
    sDG[0] = sMI[0] = sGD[0] = sIM[0] = -FLT_MAX;
    const float* qt1 = q_tr + (size_t)(i - 1) * 7;
    const float* qt0 = q_tr + (size_t)i * 7;
    const float q_m2m = qt1[M2M], q_m2d = qt1[M2D], q_d2m = qt1[D2M], q_d2d = qt1[D2D],
                q_i2m = qt1[I2M], q_i2i = qt0[I2I], q_m2i = qt0[M2I];
    const int find_max = (local || i == Lq);
    const float* qp = q_p + (size_t)i * 20;
    const float* ssrow = use_ss ? S33 + (size_t)q_ss[i] * 44 : NULL;
    float mm = 0.0f;
    for (int j = 1; j <= Lt; ++j) {
      const float* tt1 = t_tr + (size_t)(j - 1) * 7;
      const float* tt0 = t_tr + (size_t)j * 7;
      const float t_m2m = tt1[M2M], t_m2d = tt1[M2D], t_d2m = tt1[D2M], t_d2d = tt1[D2D],
                  t_i2m = tt1[I2M], t_i2i = tt0[I2I], t_m2i = tt0[M2I];
      unsigned b = 0;
      float c;
      /* 5-way max with strict '>' and first-wins ties, :241-273 */
      c = (dMM + q_m2m) + t_m2m;
      if (c > smin) b = ST_MM;
      mm = (smin > c) ? smin : c;           /* _mm256_max_ps(smin, c) */
      c = (dGD + q_m2m) + t_d2m;
      if (c > mm) b = ST_GD;
      mm = (mm > c) ? mm : c;
      c = (dIM + q_i2m) + t_m2m;
      if (c > mm) b = ST_IM;
      mm = (mm > c) ? mm : c;
      c = (dDG + q_d2m) + t_m2m;
      if (c > mm) b = ST_DG;
      mm = (mm > c) ? mm : c;
      c = (dMI + q_m2m) + t_i2m;
      if (c > mm) b = ST_MI;
      mm = (mm > c) ? mm : c;
      float Si = log2f4_scalar(dot20(qp, t_p + (size_t)j * 20));   /* :277 */
      if (use_ss) Si = (ssw * ssrow[t_ss[j]]) + Si;                /* :210,279 */
      Si = Si + shift;                                             /* :281 */
      mm = mm + Si;
      const float lMM = sMM[j - 1], lGD = sGD[j - 1], lIM = sIM[j - 1];
      const float uMM = sMM[j], uDG = sDG[j], uMI = sMI[j];
      dMM = sMM[j]; dDG = sDG[j]; dMI = sMI[j]; dGD = sGD[j]; dIM = sIM[j];   /* :294-298 */
      float a1, a2, gd, im, dg, mi;
      a1 = lMM + t_m2d; a2 = lGD + t_d2d;                          /* :307-315 */
      if (a1 > a2) b |= 8;
      gd = (a1 > a2) ? a1 : a2;
      a1 = (lMM + q_m2i) + t_m2m; a2 = (lIM + q_i2i) + t_m2m;      /* :324-332 */
      if (a1 > a2) b |= 16;
      im = (a1 > a2) ? a1 : a2;
      a1 = uMM + q_m2d; a2 = uDG + q_d2d;                          /* :340-348 */
      if (a1 > a2) b |= 32;
      dg = (a1 > a2) ? a1 : a2;
      a1 = (uMM + q_m2m) + t_m2i; a2 = (uMI + q_m2m) + t_i2i;      /* :358-366 */
      if (a1 > a2) b |= 64;
      mi = (a1 > a2) ? a1 : a2;
      if (celloff && celloff[(size_t)i * (Lt + 1) + j]) {          /* :373-392 */
        mm = mm + -FLT_MAX; gd = gd + -FLT_MAX; im = im + -FLT_MAX;
        dg = dg + -FLT_MAX; mi = mi + -FLT_MAX;
      }
      sMM[j] = mm; sDG[j] = dg; sMI[j] = mi; sGD[j] = gd; sIM[j] = im;        /* :396-400 */
      if (bt) bt[(size_t)i * (Lt + 1) + j] = (uint8_t)b;                      /* :403-417 */
      if (find_max && mm > best) { best = mm; bi = i; bj = j; }               /* :423-455 */
    }
    if (!local && mm > best) { best = mm; bi = i; bj = Lt; }                  /* :462-486 */
  }
  free(sMM);
  *score = best; *i2 = bi; *j2 = bj;
  return 0;
}

/* Follows Viterbi::Backtrace, src/hhviterbi.cpp:83-160. Arrays need i2+j2+2 entries; entry 0 unused.
 * Returns nsteps; step 1 = (i2,j2). */
int hho_backtrace(int Lt, const uint8_t* bt, int i2, int j2, int* i_steps, int* j_steps,
                  uint8_t* states, int* matched_cols) {
  int step = 0, i = i2, j = j2, mc = 0;
  int state = ST_MM;
  while (state != ST_STOP) {
    ++step;
    states[step] = (uint8_t)state; i_steps[step] = i; j_steps[step] = j;
    const uint8_t c = bt[(size_t)i * (Lt + 1) + j];
    switch (state) {
      case ST_MM: ++mc; state = (i <= 1 || j <= 1) ? ST_STOP : (c & 7); --i; --j; break;
      case ST_GD: if (j <= 1) state = ST_STOP; else { if (c & 8) state = ST_MM; --j; } break;
      case ST_IM: if (j <= 1) state = ST_STOP; else { if (c & 16) state = ST_MM; --j; } break;
      case ST_DG: if (i <= 1) state = ST_STOP; else { if (c & 32) state = ST_MM; --i; } break;
      case ST_MI: if (i <= 1) state = ST_STOP; else { if (c & 64) state = ST_MM; --i; } break;
      default: state = ST_STOP; break;
    }
  }
  states[step] = ST_MM;
  *matched_cols = mc;
  return step;
}

/* Follows Viterbi::ExcludeAlignment, src/hhviterbi.cpp:61-77 (cross of half-width 40 around each
 * path step 1 <= step < nsteps). celloff: u8[(Lq+1)*(Lt+1)], set to 1. */
void hho_exclude_alignment(int Lq, int Lt, const int* i_steps, const int* j_steps, int nsteps,
                           uint8_t* celloff) {
  const int W = 40; /* VITERBI_PATH_WIDTH, src/hhdecl.h:50 */
  for (int s = 1; s < nsteps; ++s) {
    const int i = i_steps[s], j = j_steps[s];
    for (int ii = (i - W > 1 ? i - W : 1); ii <= (i + W < Lq ? i + W : Lq); ++ii)
      celloff[(size_t)ii * (Lt + 1) + j] = 1;
    for (int jj = (j - W > 1 ? j - W : 1); jj <= (j + W < Lt ? j + W : Lt); ++jj)
      celloff[(size_t)i * (Lt + 1) + jj] = 1;
  }
}

/* ------------------------------------------------------------------ prefilter */

/* Follows flog2, src/util-inl.h:83-93 (note the double-precision polynomial constants). */
static inline float flog2_scalar(float x) {
  if (x <= 0) return -128;
  uint32_t u = f2u(x);
  float e = (float)((int)((u & 0x7F800000u) >> 23) - 0x7f);
  x = u2f((u & 0x007FFFFFu) | 0x3f800000u);
  x -= 1.0;
  x *= (1.441740 + x * (-0.7077702 + x * (0.4123442 + x * (-0.1903190 + x * 0.0440047))));
  return x + e;
}
float hho_flog2(float x) { return flog2_scalar(x); }

/* Linear (un-striped) query profile. Follows Prefilter::stripe_query_profile,
 * src/hhprefilter.cpp:356-424: prof[k*Lq + pos] for k<219 from q.p[pos] (0-based pos indexing the
 * 1-based p array: SURVEY App. D-4), row 219 = ANY state = offset-1.
 *   q_p: (Lq+2)*20, q_pav: 20, lib: 219*20 linear column-state probabilities. */
void hho_prefilter_query_profile(int Lq, const float* q_p, const float* q_pav, const float* lib,
                                 int score_offset, int bit_factor, uint8_t* prof) {
  for (int k = 0; k < 219; ++k)
    for (int pos = 0; pos < Lq; ++pos) {
      float sum = 0;
      for (int a = 0; a < 20; ++a) sum += ((q_p[(size_t)pos * 20 + a] * lib[k * 20 + a]) / q_pav[a]);
      float dummy = flog2_scalar(sum) * bit_factor + score_offset + 0.5;
      uint8_t v;
      if (dummy > 255.0) v = 255; else if (dummy < 0) v = 0; else v = (uint8_t)dummy;
      prof[(size_t)k * Lq + pos] = v;
    }
  for (int pos = 0; pos < Lq; ++pos) prof[(size_t)219 * Lq + pos] = (uint8_t)(score_offset - 1);
}

/* Follows Prefilter::ungapped_sse_score, src/hhprefilter.cpp:214-275, un-striped:
 * S(i,j) = max(0, min(255, S(i-1,j-1) + prof[x_j][i]) - offset); result = max over all cells.
 * Striped padding positions (i >= Lq) hold `offset` => contribute max(0, S) which never exceeds
 * the running maximum of real cells, so they are omitted. */
int hho_ungapped_score(int Lq, const uint8_t* prof, const uint8_t* dbseq, int Lt, int offset) {
  uint8_t* prev = (uint8_t*)calloc((size_t)Lq + 1, 1);
  uint8_t* cur = (uint8_t*)calloc((size_t)Lq + 1, 1);
  int smax = 0;
  for (int j = 0; j < Lt; ++j) {
    const uint8_t* row = prof + (size_t)dbseq[j] * Lq;
    for (int i = 0; i < Lq; ++i) {
      int s = (i > 0 ? prev[i - 1] : 0) + row[i];
      if (s > 255) s = 255;
      s -= offset;
      if (s < 0) s = 0;
      cur[i] = (uint8_t)s;
      if (s > smax) smax = s;
    }
    uint8_t* t = prev; prev = cur; cur = t;
  }
  free(prev); free(cur);
  return smax;
}

/* Stage-1 length correction, src/hhprefilter.cpp:477. */
int hho_ungapped_corrected(int raw, int Lq, int Lt, int bit_factor) {
  return raw - (int)(bit_factor * (flog2_scalar((float)Lq) + flog2_scalar((float)Lt)));
}

/* Follows Prefilter::swStripedByte, src/hhprefilter.cpp:70-212, for the AVX2 build (32 byte lanes,
 * segLen = ceil(Lq/32), full-width byte shift _mm256_shift_left<1>, lib/simd/simd.h:184-187): gapped local
 * SW on unsigned saturating bytes, Farrar striping with the SWPS3-style lazy-F loop that does NOT update E
 * (so the result can depend on the striping, SURVEY App. D-5 -- hence this lane-exact emulation rather than
 * a textbook SW).  prof: LINEAR profile [220][Lq]; padding positions behave as `bias` (:392-393).
 * gap_open here is the reference's gapOpen argument (= prefilter_gap_open + prefilter_gap_extend, :456). */
int hho_sw_striped_byte(int Lq, const uint8_t* prof, const uint8_t* dbseq, int Lt, int gap_open,
                        int gap_extend, int bias) {
  enum { V = 32 };
  const int W = (Lq + V - 1) / V;
  uint8_t* buf = (uint8_t*)calloc((size_t)3 * W * V, 1);
  uint8_t *Hst = buf, *Hld = buf + (size_t)W * V, *E = buf + (size_t)2 * W * V;
  int vmax[V];
  for (int k = 0; k < V; ++k) vmax[k] = 0;
#define SUBS(a, b) ((a) > (b) ? (a) - (b) : 0)
  for (int i = 0; i < Lt; ++i) {
    int vF[V], vH[V], vMaxCol[V];
    const uint8_t* row = prof + (size_t)dbseq[i] * Lq;
    for (int k = 0; k < V; ++k) { vF[k] = 0; vMaxCol[k] = 0; }
    for (int k = V - 1; k > 0; --k) vH[k] = Hst[(size_t)(W - 1) * V + k - 1];   /* shiftl(pvHStore[segLen-1]) */
    vH[0] = 0;
    { uint8_t* t = Hld; Hld = Hst; Hst = t; }
    for (int j = 0; j < W; ++j) {
      for (int k = 0; k < V; ++k) {
        const int pos = k * W + j;
        const int p = pos < Lq ? row[pos] : bias;
        int h = vH[k] + p; if (h > 255) h = 255;
        h = SUBS(h, bias);
        int e = E[(size_t)j * V + k];
        if (e > h) h = e;
        if (vF[k] > h) h = vF[k];
        if (h > vMaxCol[k]) vMaxCol[k] = h;
        Hst[(size_t)j * V + k] = (uint8_t)h;
        h = SUBS(h, gap_open);
        e = SUBS(e, gap_extend);
        if (h > e) e = h;
        E[(size_t)j * V + k] = (uint8_t)e;
        int f = SUBS(vF[k], gap_extend);
        if (h > f) f = h;
        vF[k] = f;
        vH[k] = Hld[(size_t)j * V + k];
      }
    }
    /* lazy F */
    int j = 0;
    for (int k = V - 1; k > 0; --k) vF[k] = vF[k - 1];
    vF[0] = 0;
    for (;;) {
      int all = 1;
      for (int k = 0; k < V; ++k) {
        const int h = Hst[(size_t)j * V + k];
        if (SUBS(vF[k], SUBS(h, gap_open)) != 0) all = 0;
      }
      if (all) break;
      for (int k = 0; k < V; ++k) {
        int h = Hst[(size_t)j * V + k];
        if (vF[k] > h) h = vF[k];
        if (h > vMaxCol[k]) vMaxCol[k] = h;
        Hst[(size_t)j * V + k] = (uint8_t)h;
        vF[k] = SUBS(vF[k], gap_extend);
      }
      if (++j >= W) {
        j = 0;
        for (int k = V - 1; k > 0; --k) vF[k] = vF[k - 1];
        vF[0] = 0;
      }
    }
    for (int k = 0; k < V; ++k) if (vMaxCol[k] > vmax[k]) vmax[k] = vMaxCol[k];
  }
#undef SUBS
  int score = 0;
  for (int k = 0; k < V; ++k) if (vmax[k] > score) score = vmax[k];
  free(buf);
  return score;
}

/* Follows fpow2, src/util-inl.h:190-214. */
float hho_fpow2(float x) {
  if (x >= FLT_MAX_EXP) return FLT_MAX;
  if (x <= FLT_MIN_EXP) return 0.0f;
  float tx = (x - 0.5f) + (3 << 22);
  int lx = (int)(f2u(tx) - 0x4b400000u);
  float dx = x - (float)lx;
  x = 1.0f + dx * (0.693019f + dx * (0.241404f + dx * (0.0520749f + dx * 0.0134929f)));
  return u2f(f2u(x) + ((uint32_t)lx << 23));
}

/* ------------------------------------------------------------------------------------------------
 * HHM text -> DP inputs: HMM::Read (src/hhhmm.cpp:202-691) and the query-independent part of
 * PrepareTemplateHMM (src/hhfunc.cpp:165-188).
 * ---------------------------------------------------------------------------------------------- */

/* fast_log2, src/util-inl.h:108-128.  The table is the one a real run ends up with: the first caller is
 * HMM::AddTransitionPseudocounts in hhhmm.cpp, where log(float) binds to the double-precision C log. */
static float g_lg2[1025], g_diff[1025];
static int g_lg2_ready = 0;
float hho_fast_log2(float x) {
  if (x <= 0) return -100000;
  if (!g_lg2_ready) {
    float prev = 0.0f;
    g_lg2[0] = 0.0f;
    for (int i = 1; i <= 1024; ++i) {
      g_lg2[i] = (float)(log((double)(float)(1024 + i)) * 1.442695041 - (double)10.0f);
      g_diff[i - 1] = (float)((double)(g_lg2[i] - prev) * 1.2352E-4);
      prev = g_lg2[i];
    }
    g_lg2_ready = 1;
  }
  uint32_t u = f2u(x);
  int a = (int)((u & 0x7F800000u) >> 23) - 0x7f;
  int b = (int)((u & 0x007FE000u) >> 13);
  int c = (int)(u & 0x00001FFFu);
  return (float)a + g_lg2[b] + g_diff[b] * (float)c;
}

/* strinta / strint, src/util.cpp:133-196: next integer in the string ('*' -> deflt), advancing *pp;
 * *pp becomes NULL when the string holds no further integer. */
static int next_int(const char** pp, int star_ok, int deflt) {
  const char* p = *pp;
  const char* p0 = p;
  if (!p) return INT32_MIN;
  while (*p != '\0' && *p != '\n' && !(*p >= '0' && *p <= '9') && !(star_ok && *p == '*')) p++;
  if (*p == '\0' || *p == '\n') { *pp = NULL; return INT32_MIN; }
  if (*p == '*') { *pp = p + 1; return deflt; }
  int neg = (p > p0 && p[-1] == '-');
  long v = 0;
  while (*p >= '0' && *p <= '9') { v = v * 10 + (*p - '0'); p++; }
  *pp = p;
  return neg ? -(int)v : (int)v;
}

/* alphabetical column order of HHM files -> internal amino-acid numbers (s2a, src/hhdecl.cpp) */
static const int kS2A[20] = {0, 4, 3, 6, 13, 7, 8, 9, 11, 10, 12, 2, 14, 5, 1, 15, 16, 19, 17, 18};

static int ss_code(char c) {   /* ss2i, src/hhutil-inl.h:123-146 */
  if (c >= 'a' && c <= 'z') c += 'A' - 'a';
  switch (c) {
    case '.': case '-': case 'X': return 0;
    case 'H': return 1;
    case 'E': return 2;
    case 'C': case '~': case 'I': return 3;
    case 'S': return 4; case 'T': return 5; case 'G': return 6; case 'B': return 7;
    case ' ': case '\t': case '\n': return -1;
  }
  return -2;
}
static char ss_norm(char c) {   /* ss2ss, src/hhutil-inl.h:217-243 */
  switch (c) {
    case '~': case 'I': return 'C';
    case 'i': return 'c';
    case 'H': case 'E': case 'C': case 'S': case 'T': case 'G': case 'B':
    case 'h': case 'e': case 'c': case 's': case 't': case 'g': case 'b': case '.': return c;
  }
  return '-';
}
static int conf_code(char c) {  /* cf2i, src/hhutil-inl.h:248-266 */
  if (c >= '0' && c <= '9') return c - '0' + 1;
  return 0;
}

static const char* next_line(const char* p, const char* end) {
  while (p < end && *p != '\n') p++;
  return p < end ? p + 1 : end;
}
static int blank_line(const char* p, const char* end) {
  for (; p < end && *p != '\n'; ++p) if (*p != ' ' && *p != '\t' && *p != '\r') return 0;
  return 1;
}

/* Parse one HHM record.  Outputs (caller-allocated, maxL columns):
 *   f_mb[(maxL+2)*20]   the column integers of the file, ALPHABETICAL amino-acid order, '*' = 99999, rows 1..L
 *   tr_mb[(maxL+1)*7]   transition integers rows 0..L, file order = enum order M2M,M2I,M2D,I2M,I2I,D2M,D2D
 *   neff_mb[(maxL+1)*3] Neff_M, Neff_I, Neff_D integers rows 0..L
 *   null_mb[20]         NULL line (alphabetical); untouched when the record has none (*has_null = 0)
 *   ss_pred/ss_conf[maxL+2]  zero-filled, then as HMM::Read fills them (:392-446)
 * Returns L (number of columns read), or <0 on malformed input. */
int hho_hhm_parse(const char* text, long len, int maxL, float* neff_hmm, int* has_pc, int* has_null,
                  int* null_mb, int* f_mb, int* tr_mb, int* neff_mb, uint8_t* ss_pred, uint8_t* ss_conf,
                  int* nss_pred_out) {
  const char* end = text + len;
  const char* p = text;
  int Lstated = 0, i = 0, nss_pred = -1, nss_conf = -1;
  *neff_hmm = 0; *has_pc = 0; *has_null = 0;
  memset(ss_pred, 0, (size_t)maxL + 2); memset(ss_conf, 0, (size_t)maxL + 2);
  while (p < end && !(p[0] == '/' && p + 1 < end && p[1] == '/')) {
    const char* line = p;
    p = next_line(p, end);
    if (blank_line(line, end)) continue;
    if (!strncmp(line, "HH", 2)) continue;
    if (!strncmp(line, "LENG", 4)) { const char* q = line + 4; Lstated = next_int(&q, 0, 0); }
    else if (!strncmp(line, "NEFF", 4) || !strncmp(line, "NAA", 3)) {   /* sscanf(line+6, "%f", &Neff_HMM), :296 */
      const char* e = line;
      while (e < end && *e != '\n') e++;
      if (e - line > 6) {
        char buf[256];
        size_t n = (size_t)(e - line - 6) < sizeof buf - 1 ? (size_t)(e - line - 6) : sizeof buf - 1;
        memcpy(buf, line + 6, n); buf[n] = 0;
        (void)sscanf(buf, "%f", neff_hmm);            /* no number: the value stays */
      }
    }
    else if (!strncmp(line, "PCT", 3)) *has_pc = 1;
    else if (!strncmp(line, "SEQ", 3)) {
      int k = -1, l = 1, m = 1;
      while (p < end && *p != '#') {
        const char* s = p;
        p = next_line(p, end);
        if (*s == '>') {
          k++;
          if (!strncmp(s, ">ss_pred", 8)) nss_pred = k;
          else if (!strncmp(s, ">ss_conf", 8)) nss_conf = k;
          l = 1; m = 1;
        } else if (k >= 0) {
          for (const char* h = s; h < end && *h != '\n' && *h > '\0'; ++h) {
            if (k == nss_pred) {
              int c0 = ss_code(*h);
              if (c0 >= 0 && c0 <= 3 && *h != '.') {
                char c = ss_norm(*h);
                if (c != '.' && !(c >= 'a' && c <= 'z') && m <= maxL) ss_pred[m++] = (uint8_t)ss_code(c);
                l++;
              }
            } else if (k == nss_conf) {
              if (*h == '-' || (*h >= '0' && *h <= '9')) { if (l <= maxL) ss_conf[l] = (uint8_t)conf_code(*h); l++; }
            }
          }
        }
      }
      if (p < end) p = next_line(p, end);   /* the '#' line */
    }
    else if (!strncmp(line, "NULL", 4)) {
      const char* q = line + 4;
      for (int a = 0; a < 20 && q; ++a) null_mb[a] = next_int(&q, 1, 99999);
      if (!q) return -3;
      *has_null = 1;
    }
    else if (!strncmp(line, "HMM", 3)) {
      p = next_line(p, end);                  /* transition labels */
      const char* q = p; p = next_line(p, end);
      for (int a = 0; a < 7 && q; ++a) tr_mb[a] = next_int(&q, 1, 99999);
      for (int a = 0; a < 3; ++a) neff_mb[a] = next_int(&q, 1, 99999);
      if (!q) return -4;
      while (p < end && !(p[0] == '/' && p[1] == '/') && p[0] != '#') {
        const char* s = p; p = next_line(p, end);
        if (blank_line(s, end)) continue;
        q = s + 1;
        (void)next_int(&q, 0, 0);             /* column number */
        ++i;
        if (i > Lstated) return -5;
        if (i > maxL) return -6;
        for (int a = 0; a < 20 && q; ++a) f_mb[i * 20 + a] = next_int(&q, 1, 99999);
        (void)next_int(&q, 0, 0);             /* l[i] */
        if (!q) return -7;
        q = p; p = next_line(p, end);
        if (*q != ' ' && *q != '\t') return -8;
        for (int a = 0; a < 7 && q; ++a) tr_mb[i * 7 + a] = next_int(&q, 1, 99999);
        for (int a = 0; a < 3; ++a) neff_mb[i * 3 + a] = next_int(&q, 1, 99999);
        if (!q) return -9;
      }
      if (p < end && p[0] == '/' && p[1] == '/') break;
    }
  }
  if (nss_pred_out) *nss_pred_out = nss_pred;
  return i;
}

typedef struct {
  float gapb, gapd, gape, gapf, gapg, gaph, gapi;   /* Parameters::gap*, src/hhdecl.cpp:74-80 */
  int pcm;                                          /* par.pc_hhm_nocontext_mode (:64) */
  float pca, pcb, pcc;                              /* par.pc_hhm_nocontext_a/b/c */
} hho_prep_params;

/* HMM::Read's number conversion + AddTransitionPseudocounts (src/hhhmm.cpp:1722-1785) + PreparePseudocounts
 * (:1811-1815) + AddAminoAcidPseudocounts (:1874-1921, modes 0..3) + CalculateAminoAcidBackground
 * (:1854-1868).  pb[20] = the background in INTERNAL order that HMM::Read leaves in the global pb after this
 * record's NULL line.  Outputs p[(L+2)*20] (pre-null-model), tr[(L+1)*7], pav[20]. */
int hho_hhm_prepare(int L, const int* f_mb, const int* tr_mb, const int* neff_mb, const float* pb,
                    float neff_hmm, int has_pc, const hho_prep_params* pp, const float* R /*[20][20]*/,
                    float* p, float* tr, float* pav) {
  float* f = (float*)malloc((size_t)(L + 2) * 20 * sizeof(float));
  float* NM = (float*)malloc((size_t)(L + 2) * 3 * sizeof(float));
  if (!f || !NM) { free(f); free(NM); return -1; }
  for (int i = 1; i <= L; ++i)
    for (int a = 0; a < 20; ++a) f[i * 20 + kS2A[a]] = hho_fpow2((float)(-f_mb[i * 20 + a]) / 1000);
  for (int a = 0; a < 20; ++a) f[a] = f[(L + 1) * 20 + a] = pb[a];
  for (int i = 0; i <= L; ++i) {
    for (int k = 0; k < 7; ++k) tr[i * 7 + k] = (float)(-tr_mb[i * 7 + k]) / 1000;
    for (int k = 0; k < 3; ++k) NM[i * 3 + k] = (float)neff_mb[i * 3 + k] / 1000;
    if (i >= 1 && NM[i * 3] == 0) NM[i * 3] = 1;
  }
  if (pp->gapb > 0) {
    float pM2D, pM2I, pM2M, pI2I, pI2M, pD2D, pD2M;
    pM2D = pM2I = (float)(pp->gapd * 0.0286);
    pM2M = 1 - pM2D - pM2I;
    pI2I = (float)(1.0 * pp->gape / (pp->gape - 1 + 1.0 / 0.75));
    pI2M = 1 - pI2I;
    pD2D = (float)(1.0 * pp->gape / (pp->gape - 1 + 1.0 / 0.75));
    pD2M = 1 - pD2D;
    const float gapb = pp->gapb;
    for (int i = 0; i <= L; ++i) {
      float* t = tr + i * 7;
      float p0 = (NM[i * 3] - 1) * hho_fpow2(t[M2M]) + gapb * pM2M;
      float p1 = (NM[i * 3] - 1) * hho_fpow2(t[M2D]) + gapb * pM2D;
      float p2 = (NM[i * 3] - 1) * hho_fpow2(t[M2I]) + gapb * pM2I;
      if (i == 0) p1 = p2 = 0;
      if (i == L) p1 = p2 = 0;
      float sum = p0 + p1 + p2 + FLT_MIN;
      t[M2M] = hho_fast_log2(p0 / sum);
      t[M2D] = hho_fast_log2(p1 / sum) * pp->gapf;
      t[M2I] = hho_fast_log2(p2 / sum) * pp->gapg;
      p0 = NM[i * 3 + 1] * hho_fpow2(t[I2M]) + gapb * pI2M;
      p1 = NM[i * 3 + 1] * hho_fpow2(t[I2I]) + gapb * pI2I;
      sum = p0 + p1 + FLT_MIN;
      t[I2M] = hho_fast_log2(p0 / sum);
      t[I2I] = hho_fast_log2(p1 / sum) * pp->gapi;
      p0 = NM[i * 3 + 2] * hho_fpow2(t[D2M]) + gapb * pD2M;
      p1 = NM[i * 3 + 2] * hho_fpow2(t[D2D]) + gapb * pD2D;
      if (i == L) p1 = 0;
      sum = p0 + p1 + FLT_MIN;
      t[D2M] = hho_fast_log2(p0 / sum);
      t[D2D] = hho_fast_log2(p1 / sum) * pp->gaph;
    }
  }
  int pcm = has_pc ? 0 : pp->pcm;
  if (pcm < 0 || pcm > 3) { free(f); free(NM); return -2; }
  for (int i = 1; i <= L; ++i) {
    const float* fi = f + i * 20;
    float tau = 0;
    if (pcm == 1) tau = pp->pca;
    else if (pcm == 2 && pp->pcc == 1.0f) tau = (float)fmin(1.0, pp->pca / (1. + NM[i * 3] / pp->pcb));
    else if (pcm == 2) tau = (float)fmin(1.0, pp->pca / (1. + powf(NM[i * 3] / pp->pcb, pp->pcc)));   /* pow(float,float) */
    else if (pcm == 3) {                                                                              /* :1911-1918 */
      float x = NM[i * 3] / pp->pcb;
      float pca3 = (float)(0.793 + 0.048 * (pp->pcb - 10.0));
      tau = (float)fmax(0.0, pca3 * (1 - x + pp->pcc * x * (1 - x)));
    }
    for (int a = 0; a < 20; ++a) {
      if (pcm == 0) { p[i * 20 + a] = fi[a]; continue; }
      /* g[i][a] = ScalarProd20(R[a], f[i]): plain left-to-right sum (SSE undefined, src/hhhit-inl.h:117) */
      const float* Ra = R + a * 20;
      float g = fi[0] * Ra[0];
      for (int b = 1; b < 20; ++b) g = g + fi[b] * Ra[b];
      p[i * 20 + a] = (float)((1. - tau) * fi[a] + tau * g);
    }
  }
  for (int a = 0; a < 20; ++a) pav[a] = pb[a] * 100.0f / neff_hmm;
  for (int i = 1; i <= L; ++i)
    for (int a = 0; a < 20; ++a) pav[a] += p[i * 20 + a];
  float sum = 0.0f;
  for (int a = 0; a < 20; ++a) sum += pav[a];
  if (sum != 0.0f) {
    float fac = (float)(1.0 / sum);
    for (int a = 0; a < 20; ++a) pav[a] *= fac;
  }
  for (int a = 0; a < 20; ++a) p[a] = p[(L + 1) * 20 + a] = pav[a];
  free(f); free(NM);
  return 0;
}

/* ------------------------------------------------------------------------------------------------
 * MAC realignment of one hit: PosteriorDecoder::realign (src/hhposteriordecoder.cpp:85-118) =
 * cell-off band around the Viterbi path (maskViterbiAlignment :207-237, FWD_BKW_PATHWITDH = 40) minus previous
 * MAC alignments (excludeMACAlignment :242-258), Forward (src/hhforwardalgorithm.cpp), Backward
 * (src/hhbackwardalgorithm.cpp), MAC DP (src/hhmacalgorithm.cpp), MAC backtrace (src/hhbacktracemac.cpp:112-210).
 * No secondary-structure term (hit.ssm2 == 0), hit.self == 0.  All double/float types and the order of every
 * product and sum follow the C++ expressions.
 *   q_tr / t_tr: LINEAR transition probabilities (HMM::Log2LinTransitionProbs, src/hhhmm.cpp:2305); the boundary
 *   rows are reset here as initializeQueryHMMTransitions (src/hhposteriordecoderrunner.cpp:145-155) and
 *   initializeForAlignment (src/hhposteriordecoder.cpp:158-167) do.
 * ---------------------------------------------------------------------------------------------- */
/* ScalarProd20 of src/hhhit-inl.h:117-122 (the non-SSE return statement): left-to-right sum */
static inline float dot20_seq(const float* qi, const float* tj) {
  float s = tj[0] * qi[0];
  for (int a = 1; a < 20; ++a) s = s + tj[a] * qi[a];
  return s;
}

/* HMM::Log2LinTransitionProbs, src/hhhmm.cpp:2311: pow(2.0f, beta * tr) with float arguments = the C library's powf */
float hho_log2lin(float x) { return powf(2.0f, 1.0f * x); }

typedef struct { double mm, gd, im, dg, mi; } hho_fb_cell;

int hho_mac_realign(int Lq, const float* q_p, const float* q_tr_in, int Lt, const float* t_p, const float* t_tr_in,
                    int local, float shift, float mact, int i1, int i2, int j1, int j2, int nsteps,
                    const int* vit_i, const int* vit_j, int excl_n, const int* excl_off, const int* excl_i,
                    const int* excl_j, int* res, float* sum_of_probs, double* pforward, int* out_i, int* out_j,
                    uint8_t* out_states, float* out_post_steps, float* post /* (Lq+1)*(Lt+1) */) {
  const int W = Lt + 1;
  uint8_t* off = (uint8_t*)calloc((size_t)(Lq + 1) * W, 1);
  uint8_t* bt = (uint8_t*)calloc((size_t)(Lq + 1) * W, 1);
  float* qtr = (float*)malloc((size_t)(Lq + 1) * 7 * sizeof(float));
  float* ttr = (float*)malloc((size_t)(Lt + 1) * 7 * sizeof(float));
  hho_fb_cell* prev = (hho_fb_cell*)calloc((size_t)Lt + 3, sizeof(hho_fb_cell));
  hho_fb_cell* curr = (hho_fb_cell*)calloc((size_t)Lt + 3, sizeof(hho_fb_cell));
  double* scale = (double*)calloc((size_t)Lq + 3, sizeof(double));
  float* Sp = (float*)calloc((size_t)Lt + 2, sizeof(float));
  float* Sc = (float*)calloc((size_t)Lt + 2, sizeof(float));
  if (!off || !bt || !qtr || !ttr || !prev || !curr || !scale || !Sp || !Sc) return -1;
  memcpy(qtr, q_tr_in, (size_t)(Lq + 1) * 7 * sizeof(float));
  memcpy(ttr, t_tr_in, (size_t)(Lt + 1) * 7 * sizeof(float));
  qtr[M2D] = qtr[M2I] = qtr[I2M] = qtr[I2I] = qtr[D2M] = qtr[D2D] = 0.0f;
  { float* e = qtr + Lq * 7; e[M2M] = 1.0f; e[M2D] = e[M2I] = e[I2M] = e[I2I] = 0.0f; e[D2M] = 1.0f; e[D2D] = 0.0f; }
  ttr[M2M] = 1.0f; ttr[M2D] = ttr[M2I] = ttr[I2M] = ttr[I2I] = ttr[D2M] = ttr[D2D] = 0.0f;
  { float* e = ttr + Lt * 7; e[M2M] = 1.0f; e[M2D] = e[M2I] = e[I2M] = e[I2I] = 0.0f; e[D2M] = 1.0f; e[D2D] = 0.0f; }
#define OFF(i, j) off[(size_t)(i) * W + (j)]
#define BT(i, j) bt[(size_t)(i) * W + (j)]
#define POST(i, j) post[(size_t)(i) * W + (j)]
#define QT(i, k) qtr[(size_t)(i) * 7 + (k)]
#define TT(j, k) ttr[(size_t)(j) * 7 + (k)]
  /* band around the Viterbi path */
  for (int i = 1; i <= Lq; ++i)
    for (int j = 1; j <= Lt; ++j) OFF(i, j) = !((i < i1 && j < j1) || (i > i2 && j > j2));
  for (int s = nsteps; s >= 1; --s) {
    int lo = vit_i[s] - 40 < 1 ? 1 : vit_i[s] - 40, hi = vit_i[s] + 40 > Lq ? Lq : vit_i[s] + 40;
    for (int i = lo; i <= hi; ++i) OFF(i, vit_j[s]) = 0;
  }
  for (int s = nsteps; s >= 1; --s) {
    int lo = vit_j[s] - 40 < 1 ? 1 : vit_j[s] - 40, hi = vit_j[s] + 40 > Lt ? Lt : vit_j[s] + 40;
    for (int j = lo; j <= hi; ++j) OFF(vit_i[s], j) = 0;
  }
  for (int e = 0; e < excl_n; ++e)
    for (int k = excl_off[e]; k < excl_off[e + 1]; ++k) {
      const int i = excl_i[k], j = excl_j[k];
      for (int ii = (i - 2 < 1 ? 1 : i - 2); ii <= (i + 2 > Lq ? Lq : i + 2); ++ii) OFF(ii, j) = 1;
      for (int jj = (j - 2 < 1 ? 1 : j - 2); jj <= (j + 2 > Lt ? Lt : j + 2); ++jj) OFF(i, jj) = 1;
    }
  memset(post, 0, (size_t)(Lq + 1) * W * sizeof(float));

  /* ---- Forward */
  double pmin = local ? 1.0 : 0.0;
  const double Cshift = pow(2.0, shift);
  double scale_prod = 1.0;
  const float one = hho_fpow2(0.0f);           /* fpow2(ScoreSS) with ssm2 == 0 */
  for (int j = 1; j <= Lt; ++j) {
    if (OFF(1, j)) { memset(&curr[j], 0, sizeof(hho_fb_cell)); continue; }
    curr[j].mm = dot20_seq(q_p + 20, t_p + (size_t)j * 20) * Cshift;
    curr[j].mi = curr[j].dg = 0.0;
    curr[j].im = curr[j - 1].mm * QT(1, M2I) * TT(j - 1, M2M) + curr[j - 1].im * QT(1, I2I) * TT(j - 1, M2M);
    curr[j].gd = curr[j - 1].mm * TT(j - 1, M2D) + curr[j - 1].gd * TT(j - 1, D2D);
  }
  for (int j = 0; j <= Lt; ++j) { POST(1, j) = (float)curr[j].mm; prev[j] = curr[j]; }
  scale[0] = scale[1] = scale[2] = 1.0;
  for (int i = 2; i <= Lq; ++i) {
    if (scale_prod < DBL_MIN * 100) scale_prod = 0.0; else scale_prod *= scale[i];
    if (OFF(i, 1)) memset(&curr[1], 0, sizeof(hho_fb_cell));
    else {
      curr[1].mm = scale_prod * one * dot20_seq(q_p + (size_t)i * 20, t_p + 20) * Cshift;
      curr[1].im = curr[1].gd = 0.0;
      curr[1].mi = scale[i] * (prev[1].mm * QT(i - 1, M2M) * TT(1, M2I) + prev[1].mi * QT(i - 1, M2M) * TT(1, I2I));
      curr[1].dg = scale[i] * (prev[1].mm * QT(i - 1, M2D) + prev[1].dg * QT(i - 1, D2D));
    }
    POST(i, 1) = (float)curr[1].mm;
    double Pmax_i = 0;
    memset(curr + 2, 0, (size_t)Lt * sizeof(hho_fb_cell));
    for (int j = 2; j <= Lt; ++j) {
      if (OFF(i, j)) continue;
      curr[j].mm = dot20_seq(q_p + (size_t)i * 20, t_p + (size_t)j * 20) * Cshift * one * scale[i] *
                   (pmin + prev[j - 1].mm * QT(i - 1, M2M) * TT(j - 1, M2M) + prev[j - 1].gd * QT(i - 1, M2M) * TT(j - 1, D2M) +
                    prev[j - 1].im * QT(i - 1, I2M) * TT(j - 1, M2M) + prev[j - 1].dg * QT(i - 1, D2M) * TT(j - 1, M2M) +
                    prev[j - 1].mi * QT(i - 1, M2M) * TT(j - 1, I2M));
      curr[j].gd = (curr[j - 1].mm * TT(j - 1, M2D) + curr[j - 1].gd * TT(j - 1, D2D));
      curr[j].im = (curr[j - 1].mm * QT(i, M2I) * TT(j - 1, M2M) + curr[j - 1].im * QT(i, I2I) * TT(j - 1, M2M));
      curr[j].dg = scale[i] * (prev[j].mm * QT(i - 1, M2D) + prev[j].dg * QT(i - 1, D2D));
      curr[j].mi = scale[i] * (prev[j].mm * QT(i - 1, M2M) * TT(j, M2I) + prev[j].mi * QT(i - 1, M2M) * TT(j, I2I));
      Pmax_i = fmax(Pmax_i, curr[j].mm);
    }
    for (int j = 0; j <= Lt; ++j) POST(i, j) = (float)curr[j].mm;
    { hho_fb_cell* x = prev; prev = curr; curr = x; }
    pmin *= scale[i];
    if (pmin < DBL_MIN * 100) pmin = 0.0;
    scale[i + 1] = 1.0 / (Pmax_i + 1.0);
  }
  double Pf;
  if (local) {
    Pf = 1.0;
    for (int i = 1; i <= Lq; ++i) {
      for (int j = 1; j <= Lt; ++j) Pf += POST(i, j);
      Pf *= scale[i + 1];
    }
  } else {
    Pf = 0.0;
    for (int i = 1; i < Lq; ++i) Pf = (Pf + POST(i, Lt) * scale[i + 1]);
    for (int j = 1; j <= Lt; ++j) Pf += POST(Lq, j);
    Pf *= scale[Lq + 1];
  }
  *pforward = Pf;

  /* ---- Backward, posterior = F * B / Pforward written over the forward values */
  scale_prod = scale[Lq + 1];
  for (int j = Lt; j >= 1; --j) {
    if (OFF(Lq, j)) { POST(Lq, j) = 0.0f; prev[j].mm = 0.0; }
    else { prev[j].mm = scale[Lq + 1]; POST(Lq, j) = (float)(POST(Lq, j) * scale[Lq + 1] / Pf); }
    prev[j].mi = prev[j].dg = 0.0;
  }
  pmin = local ? scale[Lq + 1] : 0.0;
  for (int i = Lq - 1; i >= 1; --i) {
    scale_prod *= scale[i + 1];
    if (scale_prod < DBL_MIN * 100) scale_prod = 0.0;
    if (OFF(i, Lt)) { POST(i, Lt) = 0.0f; curr[Lt].mm = 0.0; }
    else { curr[Lt].mm = scale_prod; POST(i, Lt) = (float)(POST(i, Lt) * scale_prod / Pf); }
    pmin *= scale[i + 1];
    if (pmin < DBL_MIN * 100) pmin = 0.0;
    curr[Lt].im = curr[Lt].mi = curr[Lt].dg = curr[Lt].gd = 0.0;
    if (Lt > 1) memset(curr + 1, 0, (size_t)(Lt - 1) * sizeof(hho_fb_cell));
    for (int j = Lt - 1; j >= 1; --j) {
      if (OFF(i, j)) continue;
      const double pmatch = prev[j + 1].mm * dot20_seq(q_p + (size_t)(i + 1) * 20, t_p + (size_t)(j + 1) * 20) * one *
                            Cshift * scale[i + 1];
      curr[j].mm = (+pmin + pmatch * QT(i, M2M) * TT(j, M2M) + curr[j + 1].gd * TT(j, M2D) +
                    curr[j + 1].im * QT(i, M2I) * TT(j, M2M) + prev[j].dg * QT(i, M2D) * scale[i + 1] +
                    prev[j].mi * QT(i, M2M) * TT(j, M2I) * scale[i + 1]);
      curr[j].gd = (+pmatch * QT(i, M2M) * TT(j, D2M) + curr[j + 1].gd * TT(j, D2D));
      curr[j].im = (+pmatch * QT(i, I2M) * TT(j, M2M) + curr[j + 1].im * QT(i, I2I) * TT(j, M2M));
      curr[j].dg = (+pmatch * QT(i, D2M) * TT(j, M2M) + prev[j].dg * QT(i, D2D) * scale[i + 1]);
      curr[j].mi = (+pmatch * QT(i, M2M) * TT(j, I2M) + prev[j].mi * QT(i, M2M) * TT(j, I2I) * scale[i + 1]);
    }
    for (int j = 1; j <= Lt - 1; ++j) POST(i, j) *= (float)(curr[j].mm / Pf);
    { hho_fb_cell* x = prev; prev = curr; curr = x; }
  }

  /* ---- MAC dynamic programming (float) */
  float score_MAC = -FLT_MAX;
  int mi2 = 0, mj2 = 0;
  for (int j = 0; j <= Lt; ++j) Sp[j] = 0.0f;
  BT(0, 0) = 0;
  for (int i = 1; i <= Lq; ++i) {
    Sc[0] = 0.0f;
    for (int j = 1; j <= Lt; ++j) {
      if (OFF(i, j)) { Sc[j] = -FLT_MIN; BT(i, j) = ST_STOP; continue; }
      const float term1 = POST(i, j) - mact;
      const float term2 = Sp[j - 1] + POST(i, j) - mact;
      const float term3 = (float)(Sp[j] - 0.5 * mact);
      const float term4 = (float)(Sc[j - 1] - 0.5 * mact);
      float mx; uint8_t st;
      if (term1 > term2) { mx = term1; st = ST_STOP; } else { mx = term2; st = ST_MM; }
      if (term3 > mx) { mx = term3; st = ST_MI; }
      if (term4 > mx) { mx = term4; st = ST_IM; }
      Sc[j] = mx; BT(i, j) = st;
      if (mx > score_MAC && (local || i == Lq)) { mi2 = i; mj2 = j; score_MAC = mx; }
    }
    if (!local && Sc[Lt] > score_MAC) { mi2 = i; mj2 = Lt; score_MAC = Sc[Lt]; }
    for (int j = 0; j <= Lt; ++j) Sp[j] = Sc[j];
  }

  /* ---- MAC backtrace */
  for (int i = 0; i <= Lq; ++i) BT(i, 1) = ST_STOP;
  for (int j = 1; j <= Lt; ++j) BT(1, j) = ST_STOP;
  int matched = 1, step = 0, i = mi2, j = mj2;
  uint8_t state = ST_MM;
  if (BT(i, j) != ST_MM) {
    out_i[0] = i; out_j[0] = j;
  } else {
    while (state != ST_STOP) {
      ++step;
      out_states[step] = state = BT(i, j);
      out_i[step] = i; out_j[step] = j;
      if (state == ST_MM) matched++;
      if (state == ST_MM) { i--; j--; }
      else if (state == ST_IM) j--;
      else if (state == ST_MI) i--;
    }
  }
  res[0] = out_i[step]; res[1] = mi2; res[2] = out_j[step]; res[3] = mj2; res[4] = step; res[5] = matched;
  if (step) out_states[step] = ST_MM;
  float sum = 0.0f;                             /* Hit::sum_of_probs is a float accumulator (src/hhhit.h:97) */
  for (int s = 1; s <= step; ++s) {
    if (out_states[s] == ST_MM) { out_post_steps[s] = POST(out_i[s], out_j[s]); sum += out_post_steps[s]; }
    else out_post_steps[s] = 0.0f;
  }
  *sum_of_probs = sum;
#undef OFF
#undef BT
#undef POST
#undef QT
#undef TT
  free(off); free(bt); free(qtr); free(ttr); free(prev); free(curr); free(scale); free(Sp); free(Sc);
  return step;
}
