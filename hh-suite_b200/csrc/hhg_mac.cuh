// hhg_mac.cuh -- MAC realignment of the reported hits (SURVEY §8f-3), the step right after Viterbi:
//   PosteriorDecoder::realign            src/hhposteriordecoder.cpp:85-118
//   maskViterbiAlignment / excludeMAC    src/hhposteriordecoder.cpp:207-258   (cell-off band, FWD_BKW_PATHWITDH)
//   forwardAlgorithm                     src/hhforwardalgorithm.cpp:10-220    (double, row scaling)
//   backwardAlgorithm                    src/hhbackwardalgorithm.cpp:10-140   (posterior = F*B/Pforward, float store)
//   macAlgorithm                         src/hhmacalgorithm.cpp:17-160        (float DP over posteriors - mact)
//   backtraceMAC                         src/hhbacktracemac.cpp:112-210
//
// One warp per hit.  Every value is produced by the same sequence of IEEE operations as in the reference (same
// types, same association, no FMA contraction), so the posterior matrix, Pforward and the MAC path are
// bit-identical -- the parallelism comes only from what is independent in the recurrences:
//   * within a row, MM / DG / MI depend on the previous row only  -> lanes = columns
//   * GD and IM are first-order recurrences along the row          -> two lanes scan the row sequentially
//   * the row maximum (scale factors) is order-independent         -> warp reduction
//   * hits are independent                                         -> one warp each, all hits of a query (or of a
//                                                                     batch of queries, MacArgs.req_q) concurrently
// No secondary-structure term (hit.ssm2 == 0) and no self-alignment mode.
#pragma once
#include <cfloat>
#include <climits>
#include <cstdint>

namespace hhg {

struct MacHitOut {          // mirrors hhg_mac_hit (include/hhg.h)
  int32_t i1, i2, j1, j2, nsteps, matched_cols;
  float sum_of_probs;
  int32_t flags;
  double pforward;
  long long path_off;
};

struct MacArgs {
  int n, Lq, local;
  float mact;
  double Cshift;                       // pow(2.0, shift), host-computed (libm)
  const float* q_p;                    // [(Lq+2)*20]
  const float* q_tr;                   // [(Lq+1)*7] linear, boundary rows already reset
  const ColRec* cols;                  // prepared shard records
  const long long* rec0;               // [n] first record of the request's target
  const int* Lt;                       // [n]
  const float* t_tr;                   // linear template transitions, request r at tr_off[r], (Lt+1)*7 floats
  const long long* tr_off;
  const int* vit;                      // [n*5] i1,i2,j1,j2,nsteps
  const long long* vit_off;            // [n+1] into vit_i/vit_j (entries 0..nsteps-1 = steps 1..nsteps)
  const int* vit_i; const int* vit_j;
  const long long* excl_off;           // [n+1] or nullptr
  const int* excl_i; const int* excl_j;
  // -excl / -template_excl ranges (PosteriorDecoder::exclude_regions / exclude_template_regions,
  // src/hhposteriordecoder.cpp:120-152): nq query-row ranges then nt template-column ranges, {lo..., hi...} each
  int reg_nq, reg_nt;
  const int* reg;                      // [2*nq + 2*nt] = q_lo[nq], q_hi[nq], t_lo[nt], t_hi[nt] or nullptr
  // scratch / outputs
  const long long* cell_off;           // [n] offset of the request's (Lq+1)*(Lt+1) cell block
  float* post; uint8_t* off; uint8_t* bt;
  const long long* row_off;            // [n] offset (in doubles) of 10*(Lt+3) row buffers
  double* rows;
  int band_scan;                       // default 1 (HHG_MAC_BANDSCAN=0 disables): scans visit only [first, last] active column of a row
  const int* req_map;                  // optional: blockIdx.x -> request (launches over a subset of the requests)
  long long* dbg;                      // optional [n*12] per-phase clock64 totals (HHG_MAC_TIMING)
  int smem_rows;                       // bytes of dynamic shared memory available for the row buffers
  double* scale;                       // [n*(Lq+3)], or per request at scale_off (query batch)
  MacHitOut* out;
  long long* path_off;                 // [n] into out_i/out_j/out_states/out_post
  int* out_i; int* out_j; uint8_t* out_states; float* out_post;
  // query batch: request r realigns query req_q[r], of length q_L[q] with p at q_p + q_p_off[q] and transitions at
  // q_tr + q_tr_off[q]; its scale factors sit at scale + scale_off[r].  req_q == nullptr (the zero value): every
  // request uses the one query Lq / q_p / q_tr, scale factors at scale + r*(Lq+3).
  const int* req_q;                    // [n] or nullptr
  const int* q_L;                      // [nq]
  const long long* q_p_off;            // [nq]
  const long long* q_tr_off;           // [nq]
  const long long* scale_off;          // [n]
};

struct MacQuery {
  int Lq;
  const float* p;                      // [(Lq+2)*20]
  const float* tr;                     // [(Lq+1)*7]
  double* scale;                       // [Lq+3]
};

__device__ __forceinline__ MacQuery mac_query(const MacArgs& A, int r) {
  if (!A.req_q) return MacQuery{A.Lq, A.q_p, A.q_tr, A.scale + (size_t)r * (A.Lq + 3)};
  const int q = A.req_q[r];
  return MacQuery{A.q_L[q], A.q_p + A.q_p_off[q], A.q_tr + A.q_tr_off[q], A.scale + A.scale_off[r]};
}

__device__ __forceinline__ float mac_dot20(const float* __restrict__ qi, const float* __restrict__ tj) {
  float s = __fmul_rn(tj[0], qi[0]);                 // ScalarProd20, src/hhhit-inl.h:117-122: left to right
#pragma unroll
  for (int a = 1; a < 20; ++a) s = __fadd_rn(s, __fmul_rn(tj[a], qi[a]));
  return s;
}

// Gather the log2 transition rows of the requested templates from the shard's column records into (Lt+1) x 7
// arrays (enum order M2M,M2I,M2D,I2M,I2I,D2M,D2D).  The host then applies HMM::Log2LinTransitionProbs
// (src/hhhmm.cpp:2305-2313: pow(2.0f, tr) = the C library's powf, whose rounding a device function cannot reproduce)
// and the boundary rows of initializeForAlignment (src/hhposteriordecoder.cpp:158-167).
__global__ void k_mac_gather_tr(int n, const ColRec* __restrict__ cols, const long long* __restrict__ rec0,
                                const int* __restrict__ Lt, const long long* __restrict__ tr_off,
                                float* __restrict__ t_tr) {
  const int r = blockIdx.y;
  if (r >= n) return;
  const int L = Lt[r];
  float* tr = t_tr + tr_off[r];
  const ColRec* c = cols + rec0[r];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i <= L; i += gridDim.x * blockDim.x) {
    float v[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (i >= 1 && i < L) {
      // row i: M2M,M2D,D2M,D2D,I2M sit in the record of column i+1 (index i), I2I,M2I in that of column i (index i-1)
      v[0] = c[i].m2m; v[1] = c[i - 1].m2i; v[2] = c[i].m2d; v[3] = c[i].i2m; v[4] = c[i - 1].i2i; v[5] = c[i].d2m;
      v[6] = c[i].d2d;
    }
#pragma unroll
    for (int k = 0; k < 7; ++k) tr[(size_t)i * 7 + k] = v[k];
  }
}

// Cell-off band: block per request.
__global__ void __launch_bounds__(256) k_mac_band(const MacArgs A) {
  const int r = blockIdx.x;
  const int Lq = mac_query(A, r).Lq, Lt = A.Lt[r], W = Lt + 1;
  uint8_t* off = A.off + A.cell_off[r];
  const int i1 = A.vit[r * 5], i2 = A.vit[r * 5 + 1], j1 = A.vit[r * 5 + 2], j2 = A.vit[r * 5 + 3], ns = A.vit[r * 5 + 4];
  const long long total = (long long)(Lq + 1) * W;
  for (long long c = threadIdx.x; c < total; c += blockDim.x) {
    const int i = (int)(c / W), j = (int)(c - (long long)i * W);
    off[c] = (i >= 1 && j >= 1) ? (uint8_t)!((i < i1 && j < j1) || (i > i2 && j > j2)) : (uint8_t)0;
  }
  __syncthreads();
  const int* vi = A.vit_i + A.vit_off[r];
  const int* vj = A.vit_j + A.vit_off[r];
  // switch on the +-40 cross around every step of the Viterbi path (idempotent stores of 0: order-free)
  for (int t = threadIdx.x; t < ns * 81; t += blockDim.x) {
    const int s = t / 81, d = t - s * 81 - 40;
    const int i = vi[s], j = vj[s];
    if (i + d >= 1 && i + d <= Lq) off[(size_t)(i + d) * W + j] = 0;
    if (j + d >= 1 && j + d <= Lt) off[(size_t)i * W + (j + d)] = 0;
  }
  __syncthreads();
  if (A.excl_off) {
    const int* ei = A.excl_i + A.excl_off[r];
    const int* ej = A.excl_j + A.excl_off[r];
    const int ne = (int)(A.excl_off[r + 1] - A.excl_off[r]);
    for (int t = threadIdx.x; t < ne * 5; t += blockDim.x) {
      const int s = t / 5, d = t - s * 5 - 2;
      const int i = ei[s], j = ej[s];
      if (i + d >= 1 && i + d <= Lq) off[(size_t)(i + d) * W + j] = 1;
      if (j + d >= 1 && j + d <= Lt) off[(size_t)i * W + (j + d)] = 1;
    }
  }
  if (A.reg) {                                             // whole query rows / template columns switched off
    __syncthreads();
    for (int g = 0; g < A.reg_nq; ++g) {
      const int lo = max(A.reg[g], 1), hi = min(A.reg[A.reg_nq + g], Lq);
      for (long long c = threadIdx.x; c < (long long)(hi - lo + 1) * Lt; c += blockDim.x) {
        const int i = lo + (int)(c / Lt), j = 1 + (int)(c % Lt);
        off[(size_t)i * W + j] = 1;
      }
    }
    const int* tr_ = A.reg + 2 * A.reg_nq;
    for (int g = 0; g < A.reg_nt; ++g) {
      const int lo = max(tr_[g], 1), hi = min(tr_[A.reg_nt + g], Lt);
      for (long long c = threadIdx.x; c < (long long)(hi - lo + 1) * Lq; c += blockDim.x) {
        const int j = lo + (int)(c / Lq), i = 1 + (int)(c % Lq);
        off[(size_t)i * W + j] = 1;
      }
    }
  }
}

// Forward + Pforward + Backward + MAC DP + backtrace: one warp per request.
// Row buffers live in shared memory when 10*(Lt+3) doubles fit (A.smem_rows), else in the global scratch.
// The sequential recurrences are written so that the scanning lanes execute ONE instruction stream with per-lane
// coefficients (a multiplication by 1.0 is exact, so "x*a + v*b" and "(x*a)*c + (v*b)*c" share the shape
// (x*A)*B + (v*C)*D); lanes that differ only in operands do not serialise.
__global__ void __launch_bounds__(32) k_mac_realign(const MacArgs A) {
  extern __shared__ __align__(16) unsigned char mac_smem[];
  const int r = A.req_map ? A.req_map[blockIdx.x] : (int)blockIdx.x, lane = threadIdx.x;
  const MacQuery Q = mac_query(A, r);
  const int Lq = Q.Lq, Lt = A.Lt[r], W = Lt + 1;
  const uint8_t* off = A.off + A.cell_off[r];
  uint8_t* bt = A.bt + A.cell_off[r];
  float* post = A.post + A.cell_off[r];
  const ColRec* tcol = A.cols + A.rec0[r] - 1;            // tcol[j] = record of column j (1-based)
  const float* ttr_g = A.t_tr + A.tr_off[r];
  const float* qtr = Q.tr;
  const float* q_p = Q.p;
  double* scale = Q.scale;
  const size_t RS = (size_t)Lt + 3;
  // per-warp working set: 10 row buffers (doubles), the template's linear transitions, the cell-off flags of the
  // current row.  In shared memory when it fits; the sequential scans below then never wait for global memory.
  const size_t need = 11 * RS * sizeof(double) + 7 * RS * sizeof(float) + RS;
  const bool in_smem = need <= (size_t)A.smem_rows;
  double* base = in_smem ? reinterpret_cast<double*>(mac_smem) : A.rows + A.row_off[r];
  float* ttr_s = in_smem ? reinterpret_cast<float*>(mac_smem + 11 * RS * sizeof(double)) : nullptr;
  uint8_t* offrow = in_smem ? mac_smem + 11 * RS * sizeof(double) + 7 * RS * sizeof(float)
                            : reinterpret_cast<uint8_t*>(A.rows + A.row_off[r] + 11 * RS);
  double *Pm = base, *Pg = base + RS, *Pi = base + 2 * RS, *Pd = base + 3 * RS, *Px = base + 4 * RS;
  double *Cm = base + 5 * RS, *Cg = base + 6 * RS, *Ci = base + 7 * RS, *Cd = base + 8 * RS, *Cx = base + 9 * RS;
  double* Xp = base + 10 * RS;                             // per-row addends of the Pforward lane
  const double Cshift = A.Cshift;
  const unsigned FULL = 0xffffffffu;
  if (in_smem) {
    for (int k = lane; k < (Lt + 1) * 7; k += 32) ttr_s[k] = ttr_g[k];
    __syncwarp();
  }
  const float* ttr = in_smem ? ttr_s : ttr_g;
#define OFFC(i, j) off[(size_t)(i) * W + (j)]
#define QT(i, k) qtr[(size_t)(i) * 7 + (k)]
#define TT(j, k) ttr[(size_t)(j) * 7 + (k)]
#define SWAP_ROWS() do { double* t_; t_ = Pm; Pm = Cm; Cm = t_; t_ = Pg; Pg = Cg; Cg = t_; t_ = Pi; Pi = Ci; Ci = t_; \
                         t_ = Pd; Pd = Cd; Cd = t_; t_ = Px; Px = Cx; Cx = t_; } while (0)
  enum { M2M = 0, M2I = 1, M2D = 2, I2M = 3, I2I = 4, D2M = 5, D2D = 6 };

  // Forward scan of row i (lanes 0 and 1):  GD: v = Cm[j-1]*t.M2D[j-1] + v*t.D2D[j-1]
  //                                          IM: v = Cm[j-1]*q.M2I[i]*t.M2M[j-1] + v*q.I2I[i]*t.M2M[j-1]
  // both as (x*A)*B + (v*C)*D with A,B,C,D per lane; off cells reset v to 0.
  // The addend of every chain does not depend on the chain itself, so all lanes precompute it (fwd_pre) and the scan
  // is v = pre[j] + (v*C)*D -- three FP64 instructions per column step instead of five.  Lane 2 accumulates
  // Pforward in the same stream: Pf += (float)Cm[j] in row-major order, Pf *= scale[i+1] at the end of each row
  // (src/hhforwardalgorithm.cpp:151-166), never reset.
  double Pf_acc = A.local ? 1.0 : 0.0;
  // Band-limited scans (A.band_scan): outside [jlo, jhi] every cell of the row is switched off, where the reference
  // computes exact zeros (GD = IM = 0, posterior 0 -> Pforward += 0.0 is a no-op) and every chain re-enters an active
  // run with v = 0; visiting only the active span therefore gives the same bits with ~Lt/band fewer dependent steps.
  // fwd_pre leaves the final zeros in the switched-off cells so the span can skip them.
  const bool bs = A.band_scan != 0;
  int jlo = 1, jhi = Lt;
  auto row_span = [&](int lo, int hi) {          // warp-wide first/last active column of the row just staged
    if (!bs) { jlo = 1; jhi = Lt; return; }
#pragma unroll
    for (int o = 16; o; o >>= 1) { lo = min(lo, __shfl_xor_sync(FULL, lo, o)); hi = max(hi, __shfl_xor_sync(FULL, hi, o)); }
    jlo = lo; jhi = hi;
  };
  auto fwd_pre = [&](int i) {
    const float qa = QT(i, M2I);
    for (int j = 1 + lane; j <= Lt; j += 32) {
      const double cm1 = Cm[j - 1];
      const bool dead = bs && offrow[j];
      Cg[j] = dead ? 0.0 : (cm1 * TT(j - 1, M2D));
      Ci[j] = dead ? 0.0 : (cm1 * qa) * TT(j - 1, M2M);
      Xp[j] = (double)(float)Cm[j];
    }
  };
  auto fwd_scan = [&](int i, int jfirst) {
    if (lane < 3) {
      const float qc = QT(i, I2I);
      double* __restrict__ dst = lane == 0 ? Cg : (lane == 1 ? Ci : Xp);
      const float* __restrict__ tt = ttr;
      const uint8_t* __restrict__ of = offrow;
      const int kc = lane == 0 ? D2D : M2M;
      double v = lane == 2 ? Pf_acc : 0.0;
      if (lane == 2 && jfirst == 2) v += dst[1];          // (only the local-mode value of Pf_acc is used)
      if (jfirst == 2 && lane < 2) dst[1] = 0.0;
      const int jbeg = max(jfirst, jlo), jend = jhi;
#pragma unroll 4
      for (int j = jbeg; j <= jend; ++j) {
        const float tc = tt[(j - 1) * 7 + kc];
        const float c1 = lane == 0 ? tc : (lane == 1 ? qc : 1.0f), d1 = lane == 1 ? tc : 1.0f;
        const double nv = dst[j] + (v * c1) * d1;
        v = (lane < 2 && of[j]) ? 0.0 : nv;
        dst[j] = v;
      }
      if (lane == 2) Pf_acc = v;
    }
  };

  long long tk[12] = {0,0,0,0,0,0,0,0,0,0,0,0}; long long t0_ = clock64();
#define TICK(k) do { const long long t1_ = clock64(); tk[k] += t1_ - t0_; t0_ = t1_; } while (0)
  // ------------------------------------------------------------------ Forward, row 1
  for (int j = lane; j <= Lt + 1; j += 32) { Cm[j] = Cg[j] = Ci[j] = Cd[j] = Cx[j] = 0.0; Pm[j] = Pg[j] = Pi[j] = Pd[j] = Px[j] = 0.0; }
  __syncwarp();
  {
    int lo = INT_MAX, hi = 0;
    for (int j = 1 + lane; j <= Lt; j += 32) {
      const uint8_t o = OFFC(1, j);
      offrow[j] = o;
      if (!o) { Cm[j] = (double)mac_dot20(q_p + 20, tcol[j].p) * Cshift; lo = min(lo, j); hi = max(hi, j); }
    }
    row_span(lo, hi);
  }
  __syncwarp();
  fwd_pre(1);
  __syncwarp();
  fwd_scan(1, 1);
  __syncwarp();
  for (int j = lane; j <= Lt; j += 32) post[(size_t)W + j] = (float)Cm[j];
  SWAP_ROWS();
  if (lane == 0) { scale[0] = scale[1] = scale[2] = 1.0; }
  double pmin = A.local ? 1.0 : 0.0, scale_prod = 1.0;
  __syncwarp();

  // ------------------------------------------------------------------ Forward, rows 2..Lq
  for (int i = 2; i <= Lq; ++i) {
    const double sc_i = scale[i];
    if (scale_prod < DBL_MIN * 100) scale_prod = 0.0; else scale_prod *= sc_i;
    const float* qi = q_p + (size_t)i * 20;
    const float q_m2m = QT(i - 1, M2M), q_i2m = QT(i - 1, I2M), q_d2m = QT(i - 1, D2M), q_m2d = QT(i - 1, M2D),
                q_d2d = QT(i - 1, D2D);
    double pmax = 0.0;
    int lo_ = INT_MAX, hi_ = 0;
    for (int j = 1 + lane; j <= Lt; j += 32) {
      double mm = 0.0, dg = 0.0, mi = 0.0;
      const uint8_t o = OFFC(i, j);
      offrow[j] = o;
      if (!o) {
        lo_ = min(lo_, j); hi_ = max(hi_, j);
        const float pf = mac_dot20(qi, tcol[j].p);
        if (j == 1) {
          mm = scale_prod * 1.0f * pf * Cshift;
        } else {
          mm = pf * Cshift * 1.0f * sc_i *
               (pmin + Pm[j - 1] * q_m2m * TT(j - 1, M2M) + Pg[j - 1] * q_m2m * TT(j - 1, D2M) +
                Pi[j - 1] * q_i2m * TT(j - 1, M2M) + Pd[j - 1] * q_d2m * TT(j - 1, M2M) +
                Px[j - 1] * q_m2m * TT(j - 1, I2M));
          pmax = fmax(pmax, mm);
        }
        dg = sc_i * (Pm[j] * q_m2d + Pd[j] * q_d2d);
        mi = sc_i * (Pm[j] * q_m2m * TT(j, M2I) + Px[j] * q_m2m * TT(j, I2I));
      }
      Cm[j] = mm; Cd[j] = dg; Cx[j] = mi;
    }
    row_span(lo_, hi_);
    __syncwarp();
    fwd_pre(i);
    __syncwarp();
    TICK(0);
    fwd_scan(i, 2);
    TICK(1);
#pragma unroll
    for (int o = 16; o; o >>= 1) pmax = fmax(pmax, __shfl_xor_sync(FULL, pmax, o));
    __syncwarp();
    for (int j = lane; j <= Lt; j += 32) post[(size_t)i * W + j] = (float)(j ? Cm[j] : 0.0);
    SWAP_ROWS();
    pmin *= sc_i;
    if (pmin < DBL_MIN * 100) pmin = 0.0;
    const double sc_next = 1.0 / (pmax + 1.0);           // every lane holds pmax after the reduction
    if (lane == 0) scale[i + 1] = sc_next;
    if (A.local) Pf_acc *= sc_next;                       // lane 2's copy is the live one
    __syncwarp();
    TICK(2);
  }

  // ------------------------------------------------------------------ Pforward
  double Pf = 0.0;
  if (A.local) {
    Pf = Pf_acc;                                          // accumulated by lane 2 during the forward scans
  } else if (lane == 2) {                                 // global mode: last column and last row only (:167-173)
    for (int i = 1; i < Lq; ++i) Pf = (Pf + post[(size_t)i * W + Lt] * scale[i + 1]);
    for (int j = 1; j <= Lt; ++j) Pf += post[(size_t)Lq * W + j];
    Pf *= scale[Lq + 1];
  }
  Pf = __shfl_sync(FULL, Pf, 2);
  TICK(3);

  // ------------------------------------------------------------------ Backward
  const double sc_last = scale[Lq + 1];
  for (int j = lane; j <= Lt + 1; j += 32) { Pm[j] = Pg[j] = Pi[j] = Pd[j] = Px[j] = 0.0; Cm[j] = Cg[j] = Ci[j] = Cd[j] = Cx[j] = 0.0; }
  __syncwarp();
  for (int j = 1 + lane; j <= Lt; j += 32) {
    float* pp = post + (size_t)Lq * W + j;
    if (OFFC(Lq, j)) { *pp = 0.0f; Pm[j] = 0.0; }
    else { Pm[j] = sc_last; *pp = (float)(*pp * sc_last / Pf); }
  }
  scale_prod = sc_last;
  pmin = A.local ? sc_last : 0.0;
  __syncwarp();
  for (int i = Lq - 1; i >= 1; --i) {
    const double sc_n = scale[i + 1];
    scale_prod *= sc_n;
    if (scale_prod < DBL_MIN * 100) scale_prod = 0.0;
    pmin *= sc_n;
    if (pmin < DBL_MIN * 100) pmin = 0.0;
    const float* qn = q_p + (size_t)(i + 1) * 20;
    const float q_m2m = QT(i, M2M), q_m2i = QT(i, M2I), q_m2d = QT(i, M2D), q_i2m = QT(i, I2M), q_i2i = QT(i, I2I),
                q_d2m = QT(i, D2M), q_d2d = QT(i, D2D);
    // phase A (lanes = columns): pmatch -> Cm (scratch), DG, MI; the cell in column Lt
    int lo_ = INT_MAX, hi_ = 0;
    for (int j = 1 + lane; j <= Lt; j += 32) {
      const uint8_t o = OFFC(i, j);
      offrow[j] = o;
      if (!o) { lo_ = min(lo_, j); hi_ = max(hi_, j); }
      if (j == Lt) {
        float* pp = post + (size_t)i * W + Lt;
        if (o) { *pp = 0.0f; Cm[Lt] = 0.0; }
        else { Cm[Lt] = scale_prod; *pp = (float)(*pp * scale_prod / Pf); }
        Cg[Lt] = Ci[Lt] = Cd[Lt] = Cx[Lt] = 0.0;
      } else if (o) {
        Cm[j] = Cg[j] = Ci[j] = Cd[j] = Cx[j] = 0.0;
      } else {
        const double pmatch = Pm[j + 1] * mac_dot20(qn, tcol[j + 1].p) * 1.0f * Cshift * sc_n;
        Cd[j] = (+pmatch * q_d2m * TT(j, M2M) + Pd[j] * q_d2d * sc_n);
        Cx[j] = (+pmatch * q_m2m * TT(j, I2M) + Px[j] * q_m2m * TT(j, I2I) * sc_n);
        Cm[j] = pmatch;
        Cg[j] = (pmatch * q_m2m) * TT(j, D2M);            // addends of the GD / IM chains
        Ci[j] = (pmatch * q_i2m) * TT(j, M2M);
      }
    }
    row_span(lo_, hi_);
    __syncwarp();
    TICK(4);
    // phase B (lanes 0 and 1, right to left):  GD: v = pmatch*q.M2M*t.D2M[j] + v*t.D2D[j]
    //                                           IM: v = pmatch*q.I2M*t.M2M[j] + v*q.I2I*t.M2M[j]
    if (lane < 2) {
      double* __restrict__ dst = lane == 0 ? Cg : Ci;
      const float* __restrict__ tt = ttr;
      const uint8_t* __restrict__ of = offrow;
      const int kc = lane == 0 ? D2D : M2M;
      double v = 0.0;
      const int jbeg = min(jhi, Lt - 1), jend = max(jlo, 1);
#pragma unroll 4
      for (int j = jbeg; j >= jend; --j) {
        const float tc = tt[j * 7 + kc];
        const float c1 = lane == 0 ? tc : q_i2i, d1 = lane == 0 ? 1.0f : tc;
        const double nv = dst[j] + (v * c1) * d1;
        v = of[j] ? 0.0 : nv;
        dst[j] = v;
      }
    }
    __syncwarp();
    TICK(5);
    // phase C (lanes = columns): MM from pmatch, the finished GD / IM of column j+1 and the row below
    for (int j = 1 + lane; j <= Lt - 1; j += 32) {
      double mm = 0.0;
      if (!offrow[j]) {
        const double pmatch = Cm[j];
        mm = (+pmin + pmatch * q_m2m * TT(j, M2M) + Cg[j + 1] * TT(j, M2D) + Ci[j + 1] * q_m2i * TT(j, M2M) +
              Pd[j] * q_m2d * sc_n + Px[j] * q_m2m * TT(j, M2I) * sc_n);
      }
      Cm[j] = mm;
      post[(size_t)i * W + j] *= (float)(mm / Pf);
    }
    SWAP_ROWS();
    __syncwarp();
    TICK(6);
  }

  // ------------------------------------------------------------------ MAC dynamic programming (float)
  // S_curr[j-1] - 0.5*mact is written in double in the reference; with 0.5*mact exactly a float (halving is exact)
  // and |S| < 2^28 * 0.5*mact or S in {0, -FLT_MIN}, the difference of the two floats is exact in double, so
  // rounding it once to float equals the float subtraction used here.
  float* Sp = reinterpret_cast<float*>(base);
  float* Sc = Sp + RS;
  float* T123 = Sc + RS;                                  // best of term1..term3 per column
  uint8_t* st123 = reinterpret_cast<uint8_t*>(T123 + RS);
  __syncwarp();
  for (int j = lane; j <= Lt; j += 32) Sp[j] = 0.0f;
  const float mact = A.mact;
  const double half_mact = 0.5 * mact;
  const float half_f = (float)half_mact;
  const bool half_exact = (double)half_f == half_mact;
  float score_MAC = -FLT_MAX;
  int mi2 = 0, mj2 = 0;
  if (lane == 0) bt[0] = 0;
  __syncwarp();
  for (int i = 1; i <= Lq; ++i) {
    int lo_ = INT_MAX, hi_ = 0;
    for (int j = 1 + lane; j <= Lt; j += 32) {
      const uint8_t o = OFFC(i, j);
      offrow[j] = o;
      if (o) { if (bs) Sc[j] = -FLT_MIN; continue; }     // (bt of a switched-off cell stays STOP = 0 from the memset)
      lo_ = min(lo_, j); hi_ = max(hi_, j);
      const float p = post[(size_t)i * W + j];
      const float term1 = __fsub_rn(p, mact);
      const float term2 = __fsub_rn(__fadd_rn(Sp[j - 1], p), mact);
      const float term3 = (float)((double)Sp[j] - half_mact);
      float mx; uint8_t st;
      if (term1 > term2) { mx = term1; st = 0; } else { mx = term2; st = 2; }
      if (term3 > mx) { mx = term3; st = 6; }             // MI
      T123[j] = mx; st123[j] = st;
    }
    row_span(lo_, hi_);
    __syncwarp();
    TICK(7);
    if (lane == 0) {
      float left = jlo == 1 ? 0.0f : -FLT_MIN;            // S_curr[0] = 0; left of an active run sits a switched-off cell
      Sc[0] = 0.0f;
      uint8_t* __restrict__ btrow = bt + (size_t)i * W;
      const float* __restrict__ t123 = T123;
      const uint8_t* __restrict__ s123 = st123;
      const uint8_t* __restrict__ of = offrow;
      float* __restrict__ sc_row = Sc;
      const bool can_end = A.local || i == Lq;
#pragma unroll 4
      for (int j = jlo; j <= jhi; ++j) {
        const float t4 = half_exact ? __fsub_rn(left, half_f) : (float)((double)left - half_mact);
        float mx = t123[j]; uint8_t st = s123[j];
        if (t4 > mx) { mx = t4; st = 4; }                 // IM
        const bool o = of[j] != 0;
        mx = o ? -FLT_MIN : mx; st = o ? (uint8_t)0 : st;
        if (!o && can_end && mx > score_MAC) { mi2 = i; mj2 = j; score_MAC = mx; }
        sc_row[j] = mx; btrow[j] = st;
        left = mx;
      }
      if (!A.local && Sc[Lt] > score_MAC) { mi2 = i; mj2 = Lt; score_MAC = Sc[Lt]; }
    }
    __syncwarp();
    TICK(8);
    { float* t_ = Sp; Sp = Sc; Sc = t_; }
  }

  // ------------------------------------------------------------------ MAC backtrace (lane 0)
  if (lane == 0) {
    for (int i = 0; i <= Lq; ++i) bt[(size_t)i * W + 1] = 0;
    for (int j = 1; j <= Lt; ++j) bt[(size_t)W + j] = 0;
    const long long po = A.path_off[r];
    int* oi = A.out_i + po; int* oj = A.out_j + po; uint8_t* os = A.out_states + po; float* op = A.out_post + po;
    int matched = 1, step = 0, i = mi2, j = mj2;
    uint8_t state = 2;
    oi[0] = 0; oj[0] = 0; os[0] = 0; op[0] = 0.f;
    if (mi2 < 1 || mj2 < 1 || bt[(size_t)i * W + j] != 2) {
      oi[0] = i; oj[0] = j;
    } else {
      while (state != 0) {
        ++step;
        os[step] = state = bt[(size_t)i * W + j];
        oi[step] = i; oj[step] = j;
        if (state == 2) { matched++; i--; j--; }
        else if (state == 4) j--;
        else if (state == 6) i--;
      }
    }
    MacHitOut o;
    o.i1 = oi[step]; o.i2 = mi2; o.j1 = oj[step]; o.j2 = mj2; o.nsteps = step; o.matched_cols = matched;
    if (step) os[step] = 2;
    float sum = 0.0f;
    for (int s = 1; s <= step; ++s) {
      if (os[s] == 2) { op[s] = post[(size_t)oi[s] * W + oj[s]]; sum = __fadd_rn(sum, op[s]); }
      else op[s] = 0.0f;
    }
    o.sum_of_probs = sum; o.flags = 0; o.pforward = Pf; o.path_off = po;
    A.out[r] = o;
    TICK(9);
    if (A.dbg) for (int k = 0; k < 12; ++k) A.dbg[(size_t)r * 12 + k] = tk[k];
  }
#undef TICK
#undef OFFC
#undef QT
#undef TT
#undef SWAP_ROWS
}

}  // namespace hhg
