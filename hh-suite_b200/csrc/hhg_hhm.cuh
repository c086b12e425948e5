// hhg_hhm.cuh -- HHM text records -> device-resident column records (SURVEY §8 rows a10 + a11, §8f-1).
//
// What the reference does per target AND per query (HHEntry::getTemplateHMM -> HMM::Read, src/hhhmm.cpp:202-691,
// then PrepareTemplateHMM, src/hhfunc.cpp:165-188) is done here once per database load:
//   host  : HhmScanner      -- tokenises the text of one record into the file's integers (1/1000 bits)
//   device: k_hhm_prepare   -- thread per column: fpow2 of the emissions, transition pseudocounts
//                              (HMM::AddTransitionPseudocounts :1722-1785), g = R f (PreparePseudocounts :1811),
//                              p = (1-tau) f + tau g (AddAminoAcidPseudocounts :1874-1921) -> 112-byte ColRec
//           k_hhm_pav       -- warp per target: pav (CalculateAminoAcidBackground :1854-1868)
// Every arithmetic step keeps the reference's type and order (float vs double, unfused), so the records are
// bit-identical to what the reference's own preparation hands to Viterbi::Align.
#pragma once
#include <cfloat>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "hhg_math.cuh"

namespace hhg {

// ------------------------------------------------------------------------------------------ host: scanner
struct HhmStaging {          // one chunk of records, SoA over columns
  std::vector<int32_t> f_mb;     // [cols*20]  emission integers, file (alphabetical) order, '*' = 99999
  std::vector<int32_t> trn_mb;   // [(cols+m)*10] per row i=0..L: 7 transition integers (enum order) + Neff_M,I,D
  std::vector<uint8_t> ss;       // [cols]  ss_pred*11 + ss_conf of columns 1..L
  std::vector<int32_t> null_mb;  // [m*20]
  std::vector<float> neff_hmm;   // [m]
  std::vector<int32_t> has_pc;   // [m]
};

class HhmScanner {
 public:
  HhmScanner(const char* rec, int64_t len) : p_(rec), end_(rec + len) {
    const void* z = memchr(rec, '\0', (size_t)len);   // ffindex entries carry a trailing NUL
    if (z) end_ = (const char*)z;
  }

  // LENG and presence of a ">ss_pred" sequence, without touching the numbers.
  bool peek(int32_t* L, int32_t* has_ss) {
    *L = 0; *has_ss = 0;
    const char* p = p_;
    bool in_seq = false;
    while (p < end_) {
      const char* e = line_end(p);
      if (e - p >= 3 && !memcmp(p, "SEQ", 3)) in_seq = true;
      else if (in_seq && *p == '#') in_seq = false;
      else if (in_seq) { if (e - p >= 8 && !memcmp(p, ">ss_pred", 8)) *has_ss = 1; }
      else if (e - p >= 4 && !memcmp(p, "LENG", 4)) { const char* q = p + 4; long v; if (!integer(q, e, false, &v)) return false; *L = (int32_t)v; }
      else if (e - p >= 3 && !memcmp(p, "HMM", 3) && *L > 0) return true;   // numbers start here
      p = e < end_ ? e + 1 : end_;
    }
    return *L > 0;
  }

  // Full parse into the staging slots of this record.  Returns "" or an error description.
  std::string parse(int32_t L, int32_t* f_mb, int32_t* trn_mb, uint8_t* ss, int32_t* null_mb,
                    float* neff_hmm, int32_t* has_pc) {
    bool have_null = false, have_hmm = false;
    int pred_seq = -1, conf_seq = -1;
    std::vector<uint8_t> pred((size_t)L + 2, 0), conf((size_t)L + 2, 0);
    *neff_hmm = 0.f; *has_pc = 0;
    const char* p = p_;
    while (p < end_) {
      const char* e = line_end(p);
      const char* next = e < end_ ? e + 1 : end_;
      const size_t n = (size_t)(e - p);
      if (n >= 2 && p[0] == '/' && p[1] == '/') break;
      if (blank(p, e) || (n >= 2 && !memcmp(p, "HH", 2))) { p = next; continue; }
      if ((n >= 4 && !memcmp(p, "NEFF", 4)) || (n >= 3 && !memcmp(p, "NAA", 3))) {
        // sscanf(line+6, "%f", &Neff_HMM) (:296): a line without a number there leaves the value as it was
        if (n > 6) {
          const std::string s(p + 6, e);
          char* stop = nullptr;
          const float v = strtof(s.c_str(), &stop);
          if (stop != s.c_str()) *neff_hmm = v;
        }
      } else if (n >= 3 && !memcmp(p, "PCT", 3)) {
        *has_pc = 1;
      } else if (n >= 4 && !memcmp(p, "NULL", 4)) {
        const char* q = p + 4;
        for (int a = 0; a < 20; ++a) { long v; if (!integer(q, e, true, &v)) return "NULL line has fewer than 20 values"; null_mb[a] = (int32_t)v; }
        have_null = true;
      } else if (n >= 3 && !memcmp(p, "SEQ", 3)) {
        // displayed sequences up to the '#' line; only ss_pred / ss_conf matter for the DP (src/hhhmm.cpp:318-446)
        int k = -1, l = 1, m = 1;
        p = next;
        while (p < end_ && *p != '#') {
          e = line_end(p);
          if (*p == '>') {
            ++k; l = 1; m = 1;
            if (e - p >= 8 && !memcmp(p, ">ss_pred", 8)) pred_seq = k;
            else if (e - p >= 8 && !memcmp(p, ">ss_conf", 8)) conf_seq = k;
          } else if (k >= 0 && k == pred_seq) {
            for (const char* h = p; h < e; ++h) {
              const int code = ss_index(*h);
              if (code < 0 || code > 3 || *h == '.') continue;
              const char c = ss_canonical(*h);
              if (c != '.' && !(c >= 'a' && c <= 'z') && m <= L) pred[m++] = (uint8_t)ss_index(c);
              ++l;
            }
          } else if (k >= 0 && k == conf_seq) {
            for (const char* h = p; h < e; ++h)
              if (*h == '-' || (*h >= '0' && *h <= '9')) { if (l <= L) conf[l] = (uint8_t)(*h == '-' ? 0 : *h - '0' + 1); ++l; }
          }
          p = e < end_ ? e + 1 : end_;
        }
        e = line_end(p);
        next = e < end_ ? e + 1 : end_;
      } else if (n >= 3 && !memcmp(p, "HMM", 3)) {
        have_hmm = true;
        p = next;                                   // amino-acid labels were on the HMM line; skip transition labels
        p = skip_line(p);
        e = line_end(p);
        if (!row10(p, e, trn_mb)) return "start-state transition line is short";
        p = e < end_ ? e + 1 : end_;
        int i = 0;
        while (p < end_ && !(p[0] == '/' && p + 1 < end_ && p[1] == '/') && p[0] != '#') {
          e = line_end(p);
          if (blank(p, e)) { p = e < end_ ? e + 1 : end_; continue; }
          if (++i > L) return "more columns than LENG states";
          const char* q = p + 1;
          long v;
          if (!integer(q, e, false, &v)) return "column line without a column number";
          for (int a = 0; a < 20; ++a) { if (!integer(q, e, true, &v)) return "column line has fewer than 20 values"; f_mb[(size_t)(i - 1) * 20 + a] = (int32_t)v; }
          if (!integer(q, e, false, &v)) return "column line lacks the trailing state index";
          p = e < end_ ? e + 1 : end_;
          e = line_end(p);
          if (p >= end_ || (*p != ' ' && *p != '\t')) return "transition line missing after a column line";
          if (!row10(p, e, trn_mb + (size_t)i * 10)) return "transition line is short";
          if (trn_mb[(size_t)i * 10 + 7] == 0) trn_mb[(size_t)i * 10 + 7] = 1000;   // Neff_M == 0 -> 1 (:631-633)
          p = e < end_ ? e + 1 : end_;
        }
        if (i != L) return "fewer columns than LENG states";
        break;
      }
      p = next;
    }
    if (!have_hmm) return "no HMM section";
    if (!have_null) return "no NULL line";
    // Neff_HMM = 0 would make pav = pb*100/0 = inf and then NaN (CalculateAminoAcidBackground): refuse the record
    if (*neff_hmm == 0.f) return "Neff_HMM is 0 (no NEFF/NAA line, or NEFF 0)";
    // a record without ss_pred has no secondary structure, whatever its ss_conf says; ss_pred without ss_conf: conf 0
    for (int j = 1; j <= L; ++j) ss[j - 1] = pred_seq < 0 ? 0 : (uint8_t)(pred[j] * 11 + conf[j]);   // MAXCF = 11
    return "";
  }

 private:
  const char* p_;
  const char* end_;
  const char* line_end(const char* p) const { const void* e = memchr(p, '\n', (size_t)(end_ - p)); return e ? (const char*)e : end_; }
  const char* skip_line(const char* p) const { const char* e = line_end(p); return e < end_ ? e + 1 : end_; }
  static bool blank(const char* p, const char* e) { for (; p < e; ++p) if (*p != ' ' && *p != '\t' && *p != '\r') return false; return true; }
  // strint / strinta (src/util.cpp:133-196): next run of digits, '-' directly before it negates, '*' = 99999
  static bool integer(const char*& q, const char* e, bool star, long* out) {
    const char* start = q;
    while (q < e && !(*q >= '0' && *q <= '9') && !(star && *q == '*')) ++q;
    if (q >= e) return false;
    if (*q == '*') { ++q; *out = 99999; return true; }
    const bool neg = q > start && q[-1] == '-';
    long v = 0;
    while (q < e && *q >= '0' && *q <= '9') v = v * 10 + (*q++ - '0');
    *out = neg ? -v : v;
    return true;
  }
  static bool row10(const char* p, const char* e, int32_t* out) {
    const char* q = p;
    for (int a = 0; a < 10; ++a) { long v; if (!integer(q, e, true, &v)) return false; out[a] = (int32_t)v; }
    return true;
  }
  static int ss_index(char c) {       // ss2i, src/hhutil-inl.h:123
    if (c >= 'a' && c <= 'z') c = (char)(c - 'a' + 'A');
    switch (c) {
      case '.': case '-': case 'X': return 0;
      case 'H': return 1; case 'E': return 2;
      case 'C': case '~': case 'I': return 3;
      case 'S': return 4; case 'T': return 5; case 'G': return 6; case 'B': return 7;
      case ' ': case '\t': case '\n': return -1;
      default: return -2;
    }
  }
  static char ss_canonical(char c) {  // ss2ss, src/hhutil-inl.h:217
    switch (c) {
      case '~': case 'I': return 'C';
      case 'i': return 'c';
      case 'H': case 'E': case 'C': case 'S': case 'T': case 'G': case 'B': case '.':
      case 'h': case 'e': case 'c': case 's': case 't': case 'g': case 'b': return c;
      default: return '-';
    }
  }
};

// ------------------------------------------------------------------------------------------ device
struct HhmPrepArgs {
  float R[400];                  // R[a*20+b], PreparePseudocounts' matrix
  float gapb, gapf, gapg, gaph, gapi;
  float pM2M, pM2I, pM2D, pI2I, pI2M, pD2D, pD2M;   // a-priori transition pseudocounts (:1744-1752), host-computed
  int pcm;
  float pca, pcb, pcc;
};

// alphabetical file order (ACDEFGHIKLMNPQRSTVWY) -> internal amino-acid index (s2a, src/hhdecl.h:61) and back
#define HHG_S2A(a) ((a)==0?0:(a)==1?4:(a)==2?3:(a)==3?6:(a)==4?13:(a)==5?7:(a)==6?8:(a)==7?9:(a)==8?11:(a)==9?10: \
                    (a)==10?12:(a)==11?2:(a)==12?14:(a)==13?5:(a)==14?1:(a)==15?15:(a)==16?16:(a)==17?19:(a)==18?17:18)
#define HHG_A2S(i) ((i)==0?0:(i)==4?1:(i)==3?2:(i)==6?3:(i)==13?4:(i)==7?5:(i)==8?6:(i)==9?7:(i)==11?8:(i)==10?9: \
                    (i)==12?10:(i)==2?11:(i)==14?12:(i)==5?13:(i)==1?14:(i)==15?15:(i)==16?16:(i)==19?17:(i)==17?18:19)

// One row of HMM::AddTransitionPseudocounts (:1755-1783): tr[7] (enum order, log2) of row i of a template with L
// columns and its Neff_M / Neff_I / Neff_D, in place.
__device__ __forceinline__ void hhm_transitions_core(float* tr, float nM, float nI, float nD, int i, int L,
                                                     const HhmPrepArgs& A, const float* lg2, const float* diff) {
  if (!(A.gapb > 0.f)) return;
  const float nm1 = __fsub_rn(nM, 1.0f);
  float p0 = __fadd_rn(__fmul_rn(nm1, fpow2_dev(tr[0])), __fmul_rn(A.gapb, A.pM2M));
  float p1 = __fadd_rn(__fmul_rn(nm1, fpow2_dev(tr[2])), __fmul_rn(A.gapb, A.pM2D));
  float p2 = __fadd_rn(__fmul_rn(nm1, fpow2_dev(tr[1])), __fmul_rn(A.gapb, A.pM2I));
  if (i == 0 || i == L) p1 = p2 = 0.f;
  float sum = __fadd_rn(__fadd_rn(__fadd_rn(p0, p1), p2), FLT_MIN);
  tr[0] = fast_log2_dev(__fdiv_rn(p0, sum), lg2, diff);
  tr[2] = __fmul_rn(fast_log2_dev(__fdiv_rn(p1, sum), lg2, diff), A.gapf);
  tr[1] = __fmul_rn(fast_log2_dev(__fdiv_rn(p2, sum), lg2, diff), A.gapg);
  p0 = __fadd_rn(__fmul_rn(nI, fpow2_dev(tr[3])), __fmul_rn(A.gapb, A.pI2M));
  p1 = __fadd_rn(__fmul_rn(nI, fpow2_dev(tr[4])), __fmul_rn(A.gapb, A.pI2I));
  sum = __fadd_rn(__fadd_rn(p0, p1), FLT_MIN);
  tr[3] = fast_log2_dev(__fdiv_rn(p0, sum), lg2, diff);
  tr[4] = __fmul_rn(fast_log2_dev(__fdiv_rn(p1, sum), lg2, diff), A.gapi);
  p0 = __fadd_rn(__fmul_rn(nD, fpow2_dev(tr[5])), __fmul_rn(A.gapb, A.pD2M));
  p1 = __fadd_rn(__fmul_rn(nD, fpow2_dev(tr[6])), __fmul_rn(A.gapb, A.pD2D));
  if (i == L) p1 = 0.f;
  sum = __fadd_rn(__fadd_rn(p0, p1), FLT_MIN);
  tr[5] = fast_log2_dev(__fdiv_rn(p0, sum), lg2, diff);
  tr[6] = __fmul_rn(fast_log2_dev(__fdiv_rn(p1, sum), lg2, diff), A.gaph);
}

// the same from the integers of an HHM file (1/1000 bits; Neff * 1000)
__device__ __forceinline__ void hhm_transitions(const int32_t* __restrict__ row, int i, int L,
                                                const HhmPrepArgs& A, const float* lg2, const float* diff,
                                                float* tr) {
#pragma unroll
  for (int k = 0; k < 7; ++k) tr[k] = __fdiv_rn((float)(-row[k]), 1000.0f);
  if (!(A.gapb > 0.f)) return;
  hhm_transitions_core(tr, __fdiv_rn((float)row[7], 1000.0f), __fdiv_rn((float)row[8], 1000.0f),
                       __fdiv_rn((float)row[9], 1000.0f), i, L, A, lg2, diff);
}

// HMM::PreparePseudocounts + AddAminoAcidPseudocounts (:1811-1815, :1874-1921) of one column: f[20] -> p[20].
// tau_pre: mode 2 with pcc != 1 needs the C library's powf; the caller passes the per-column tau computed on the host.
__device__ __forceinline__ void hhm_emissions(const float* f, float nM, int pcm, const HhmPrepArgs& A, bool have_tau,
                                              float tau_pre, float* p) {
  if (pcm == 0) {
#pragma unroll
    for (int a = 0; a < 20; ++a) p[a] = f[a];
    return;
  }
  float tau = A.pca;                                                // mode 1
  if (pcm == 2 && have_tau) {
    tau = tau_pre;
  } else if (pcm == 2) {                                            // tau = fmin(1.0, pca / (1. + Neff_M[i]/pcb))
    const double den = __dadd_rn(1.0, (double)__fdiv_rn(nM, A.pcb));
    tau = __double2float_rn(fmin(1.0, __ddiv_rn((double)A.pca, den)));
  } else if (pcm == 3) {                                            // constant-diversity pseudocounts, :1911-1918
    const float x = __fdiv_rn(nM, A.pcb);
    const float pca3 = __double2float_rn(__dadd_rn(0.793, __dmul_rn(0.048, __dsub_rn((double)A.pcb, 10.0))));
    const float one_m_x = __fsub_rn(1.0f, x);
    const float inner = __fadd_rn(one_m_x, __fmul_rn(__fmul_rn(A.pcc, x), one_m_x));   // 1 - x + pcc*x*(1-x)
    tau = __double2float_rn(fmax(0.0, (double)__fmul_rn(pca3, inner)));
  }
  const double one_minus_tau = __dsub_rn(1.0, (double)tau);
#pragma unroll
  for (int a = 0; a < 20; ++a) {
    const float* Ra = A.R + a * 20;
    float g = __fmul_rn(f[0], Ra[0]);                               // ScalarProd20(R[a], f[i]), left to right
#pragma unroll
    for (int b = 1; b < 20; ++b) g = __fadd_rn(g, __fmul_rn(f[b], Ra[b]));
    p[a] = __double2float_rn(__dadd_rn(__dmul_rn(one_minus_tau, (double)f[a]), (double)__fmul_rn(tau, g)));
  }
}

// Thread per column j = 1..L of every record in the chunk.  col_off[m] are chunk-local column offsets;
// row r of record t sits at trn_mb[(col_off[t] + t + r) * 10].
__global__ void __launch_bounds__(128)
k_hhm_prepare(int m, const int* __restrict__ L, const long long* __restrict__ col_off,
              const int32_t* __restrict__ f_mb, const int32_t* __restrict__ trn_mb,
              const uint8_t* __restrict__ ss, const int32_t* __restrict__ has_pc,
              const __grid_constant__ HhmPrepArgs A, const float* __restrict__ lg2,
              const float* __restrict__ diff, ColRec* __restrict__ out, long long total_cols,
              float* __restrict__ tr_full, const float* __restrict__ tau_host) {
  // tr_full (optional): the complete transition rows tr[i][M2M,M2I,M2D,I2M,I2I,D2M,D2D], i = 0..L, of every record at
  // float offset (col_off[t] + t + i) * 7 -- what a QUERY needs (hhg_query_from_hhm); column records only keep the
  // entries the DP reads from a template
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= total_cols) return;
  int lo = 0, hi = m - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (col_off[mid] <= c) lo = mid; else hi = mid - 1;
  }
  const int t = lo, Lt = L[t];
  const int j = (int)(c - col_off[t]) + 1;
  const int32_t* rows = trn_mb + (size_t)(col_off[t] + t) * 10;
  float tr_prev[7], tr_here[7];
  hhm_transitions(rows + (size_t)(j - 1) * 10, j - 1, Lt, A, lg2, diff, tr_prev);
  hhm_transitions(rows + (size_t)j * 10, j, Lt, A, lg2, diff, tr_here);
  if (tr_full) {
    float* dst = tr_full + (size_t)(col_off[t] + t) * 7;
#pragma unroll
    for (int k = 0; k < 7; ++k) dst[(size_t)j * 7 + k] = tr_here[k];
    if (j == 1) {
#pragma unroll
      for (int k = 0; k < 7; ++k) dst[k] = tr_prev[k];
    }
  }

  float f[20];
  const int32_t* fm = f_mb + (size_t)c * 20;
#pragma unroll
  for (int a = 0; a < 20; ++a) f[HHG_S2A(a)] = fpow2_dev(__fdiv_rn((float)(-fm[a]), 1000.0f));   // :608
  const int pcm = has_pc[t] ? 0 : A.pcm;
  ColRec r;
  // pcc != 1: tau = fmin(1.0, pca / (1. + pow(Neff_M[i]/pcb, pcc))) -- the reference's pow is the C library's powf;
  // only the host's libm reproduces its bits, so tau comes precomputed per column (db_create_hhm_impl)
  hhm_emissions(f, __fdiv_rn((float)rows[(size_t)j * 10 + 7], 1000.0f), pcm, A, tau_host != nullptr,
                tau_host ? tau_host[c] : 0.f, r.p);
  r.m2m = tr_prev[0]; r.m2d = tr_prev[2]; r.d2m = tr_prev[5]; r.d2d = tr_prev[6]; r.i2m = tr_prev[3];
  r.i2i = tr_here[4]; r.m2i = tr_here[1];
  r.ss = ss ? (uint32_t)ss[c] : 0u;
  out[c] = r;
}

// Warp per record, lane a < 20 owns one amino acid: pav[a] = pb[a]*100/Neff_HMM + sum_i p[i][a] in column order,
// then NormalizeTo1 (src/util-inl.h:277-291).
__global__ void __launch_bounds__(128)
k_hhm_pav(int m, const int* __restrict__ L, const long long* __restrict__ col_off,
          const ColRec* __restrict__ cols, const int32_t* __restrict__ null_mb,
          const float* __restrict__ neff_hmm, const __grid_constant__ HhmPrepArgs A, float* __restrict__ pav,
          const float* __restrict__ pb_glob = nullptr) {
  const int t = (int)((blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (t >= m) return;
  // lane a holds internal amino acid a; find the file column that maps to it
  float acc = 0.f;
  if (lane < 20) {
    const int src = HHG_A2S(lane);
    // HHM records: HMM::Read overwrites pb[] from the file's NULL line (:543); alignments: the caller's pb
    const float pb = pb_glob ? pb_glob[lane] : fpow2_dev(__fdiv_rn((float)(-null_mb[t * 20 + src]), 1000.0f));
    acc = __fdiv_rn(__fmul_rn(pb, 100.0f), neff_hmm[t]);
    const ColRec* col = cols + col_off[t];
    const int Lt = L[t];
    int i = 0;
    for (; i + 4 <= Lt; i += 4) {
      const float v0 = col[i].p[lane], v1 = col[i + 1].p[lane], v2 = col[i + 2].p[lane], v3 = col[i + 3].p[lane];
      acc = __fadd_rn(acc, v0); acc = __fadd_rn(acc, v1); acc = __fadd_rn(acc, v2); acc = __fadd_rn(acc, v3);
    }
    for (; i < Lt; ++i) acc = __fadd_rn(acc, col[i].p[lane]);
  }
  float sum = 0.f;
#pragma unroll
  for (int a = 0; a < 20; ++a) sum = __fadd_rn(sum, __shfl_sync(0xffffffffu, acc, a));
  if (lane < 20) {
    if (sum != 0.f) acc = __fmul_rn(acc, __double2float_rn(__ddiv_rn(1.0, (double)sum)));
    pav[t * 20 + lane] = acc;
  }
}

}  // namespace hhg
