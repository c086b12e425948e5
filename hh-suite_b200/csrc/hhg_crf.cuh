// hhg_crf.cuh -- context-specific pseudocounts of the query (SURVEY §8 row a12, the default branch of PrepareQueryHMM,
// src/hhfunc.cpp:143-147, and of the prefilter profile, src/hhblits.cpp) with either engine InitializePseudocountsEngine
// (src/hhfunc.cpp:204-244) picks: the CRF of a `.crf` file, cs::CrfPseudocounts::AddToProfile
// (src/cs/crf_pseudocounts-inl.h:74-110), or the generative context library of any other file,
// cs::LibraryPseudocounts::AddToProfile (src/cs/library_pseudocounts-inl.h:58-81); then Pseudocounts::AddTo / AdmixTo
// (src/cs/pseudocounts-inl.h:41-73).
//
// Work split: the O(L * K * W * 20) part -- the context score of every state at every column, ordered double-precision
// sums -- runs in k_crf_scores / k_lib_scores; the log-sum-exp over the K = 4000 states needs exp() and log() with the bits of the
// host's C library (the reference calls libm; CUDA's double exp is a different approximation), so the O(L * K) tail
// runs on the host threads of the library.
#pragma once
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace hhg {

struct CrfHost {
  int K = 0, W = 0;                      // states, window length (odd)
  bool library = false;                  // generative context library (cs::LibraryPseudocounts), not a CRF
  std::vector<double> bias;              // [K]         CRF bias / library: log prior
  std::vector<double> w;                 // [W][20][K]  CRF context weights / library: log-probabilities; state index
                                         //             fastest (coalesced in the kernel)
  std::vector<double> pc;                // [K][20]     emission pseudocounts of the states (CRF: UpdatePseudocounts,
                                         //             library: the central column in linear space)
  std::vector<double> ww;                // [W]         library only: window weights of cs::Emission
};

// The line and number reading of the reference's serialisers (src/cs/io.h), shared by both readers.
struct TextLines {
  const char* p;
  const char* end;
  bool next(std::string& ln) {                            // cs::fgetline: trailing control characters dropped
    if (p >= end) return false;
    const char* e = (const char*)memchr(p, '\n', (size_t)(end - p));
    if (!e) e = end;
    ln.assign(p, e);
    while (!ln.empty() && (ln.back() == '\r' || ln.back() == '\0')) ln.pop_back();
    p = e < end ? e + 1 : end;
    return true;
  }
};
inline bool text_blank(const std::string& s) { for (char c : s) if ((unsigned char)c > 32) return false; return true; }
inline int text_strastoi(const char*& q, bool& ok) {     // strastoi, src/cs/io.h:76-92: '*' reads as INT_MAX
  const char* q0 = q;
  while (*q != '\0' && !(*q >= '0' && *q <= '9') && *q != '*') ++q;
  if (*q == '\0') { ok = false; return INT_MIN; }
  if (*q == '*') { ++q; return INT_MAX; }
  int i = (q > q0 && *(q - 1) == '-') ? -atoi(q) : atoi(q);
  while (*q >= '0' && *q <= '9') ++q;
  return i;
}
inline bool text_strtoi(const char*& q, int* v) {        // strtoi, src/cs/io.h:61-73
  const char* q0 = q;
  while (*q != '\0' && !(*q >= '0' && *q <= '9')) ++q;
  if (*q == '\0') return false;
  *v = (q > q0 && *(q - 1) == '-') ? -atoi(q) : atoi(q);
  while (*q >= '0' && *q <= '9') ++q;
  return true;
}
inline bool text_read_int(const std::string& ln, const char* label, int* v) {   // ReadInt, src/cs/io.h:120-131
  if (ln.find(label) == std::string::npos) return false;
  const char* q = ln.c_str() + strlen(label);             // the value follows the label at line start
  return text_strtoi(q, v);
}

// cs::Crf::Read + CrfState::Read (src/cs/crf-inl.h:56-80, crf_state-inl.h:28-76) on the text of a .crf file
inline std::string crf_parse(const char* text, int64_t len, CrfHost* out) {
  CrfHost& C = *out;
  C = CrfHost();
  TextLines in{text, text + len};
  std::string ln;
  do { if (!in.next(ln)) return "empty CRF text"; } while (text_blank(ln));
  if (ln.compare(0, 3, "CRF") != 0) return "text does not start with class id 'CRF'";
  int size = 0, wlen = 0;
  if (!in.next(ln) || !text_read_int(ln, "SIZE", &size)) return "unable to parse CRF 'SIZE'";
  if (!in.next(ln) || !text_read_int(ln, "LENG", &wlen)) return "unable to parse CRF 'LENG'";
  if (size < 1) return "CRF SIZE " + std::to_string(size) + " is not a positive number of states";
  // k_crf_scores stages the window in a 64-column shared-memory tile; the reference's reader asserts on even windows
  if (wlen < 1 || !(wlen & 1) || wlen > 63)
    return "CRF window length " + std::to_string(wlen) + " is not supported: the window must be odd and 1..63 columns";
  C.K = size; C.W = wlen;
  C.bias.assign(size, 0.0);
  C.w.assign((size_t)wlen * 20 * size, 0.0);
  C.pc.assign((size_t)size * 20, 0.0);
  for (int k = 0; k < size; ++k) {
    do { if (!in.next(ln)) return "CRF has fewer states than SIZE says"; } while (text_blank(ln));
    if (ln.compare(0, 8, "CrfState") != 0) return "state " + std::to_string(k) + " does not start with 'CrfState'";
    if (!in.next(ln)) return "truncated state";
    if (ln.find("NAME") != std::string::npos) { if (!in.next(ln)) return "truncated state"; }
    if (ln.find("BIAS") == std::string::npos) return "unable to parse CRF state 'BIAS'";
    C.bias[k] = atof(ln.c_str() + 4);
    int slen = 0, nalph = 0;
    if (!in.next(ln) || !text_read_int(ln, "LENG", &slen) || slen != wlen) return "state window length differs from the CRF's";
    if (!in.next(ln) || !text_read_int(ln, "ALPH", &nalph) || nalph != 20) return "alphabet size of a CRF state is not 20";
    if (!in.next(ln)) return "truncated state";        // alphabet description line
    double pcw[20];
    bool have_pc = false;
    int last_row = -1;
    while (in.next(ln) && !(ln.size() >= 2 && ln[0] == '/' && ln[1] == '/') ) {
      // the reference's loop condition is `buffer[0] != '/' && buffer[1] != '/'`; rows start with a digit or "PC"
      const char* q = ln.c_str();
      bool ok = true;
      if (!(ln.size() >= 2 && ln[0] == 'P' && ln[1] == 'C')) {
        int row;
        if (!text_strtoi(q, &row)) return "context weight row without a column number";
        row -= 1;
        if (row < 0 || row >= wlen) return "context weight row outside the window";
        for (int a = 0; a < 20; ++a) {
          const int v = text_strastoi(q, ok);
          if (!ok) return "context weight row has fewer than 20 values";
          C.w[((size_t)row * 20 + a) * size + k] = static_cast<double>(v) / 1000;      // kScale
        }
        last_row = row;
      } else {
        for (int a = 0; a < 20; ++a) {
          const int v = text_strastoi(q, ok);
          if (!ok) return "PC row has fewer than 20 values";
          pcw[a] = static_cast<double>(v) / 1000;
        }
        have_pc = true;
      }
    }
    if (last_row != wlen - 1) return "CRF state has the wrong number of columns";
    if (!have_pc) return "CRF state without a PC row";
    // UpdatePseudocounts (src/cs/crf_state-inl.h:137-158): the sum is a long double, log takes it as such
    double mx = -DBL_MAX;
    for (int a = 0; a < 20; ++a) if (pcw[a] > mx) mx = pcw[a];
    long double sum = 0.0;
    for (int a = 0; a < 20; ++a) sum += exp(pcw[a] - mx);
    const double tmp = mx + log(sum);
    for (int a = 0; a < 20; ++a) C.pc[(size_t)k * 20 + a] = DBL_MIN + exp(pcw[a] - tmp);
  }
  return "";
}

// cs::ContextLibrary::Read + ContextProfile::Read (src/cs/context_library-inl.h:48-68, context_profile-inl.h:80-144),
// then TransformToLog (context_profile-inl.h:213-223), on the text of a context library (.lib), and the window
// weights of cs::Emission (src/cs/emission.h:37-55): ww[c] = wcenter, ww[c +- d] = wcenter * pow(wdecay, d).
// Refusals the reference's reader does not make: even windows and windows over 63 columns, a profile LENG other than
// the library's, a row count other than LENG or a row number given twice, a row with fewer than 20 values, a negative,
// infinite or NaN PRIOR, and a value whose probability 2^(-v/1000) is 0 or infinite in double ('*' included: log 0
// turns every window with a zero count into NaN), and window weights that are not finite.
inline std::string lib_parse(const char* text, int64_t len, double wcenter, double wdecay, CrfHost* out) {
  CrfHost& C = *out;
  C = CrfHost();
  C.library = true;
  if (!std::isfinite(wcenter) || !std::isfinite(wdecay))
    return "window weights " + std::to_string(wcenter) + " / " + std::to_string(wdecay) + " are not finite";
  TextLines in{text, text + len};
  std::string ln;
  do { if (!in.next(ln)) return "empty context library text"; } while (text_blank(ln));
  if (ln.compare(0, 14, "ContextLibrary") != 0) return "text does not start with class id 'ContextLibrary'";
  int size = 0, wlen = 0;
  if (!in.next(ln) || !text_read_int(ln, "SIZE", &size)) return "unable to parse context library 'SIZE'";
  if (!in.next(ln) || !text_read_int(ln, "LENG", &wlen)) return "unable to parse context library 'LENG'";
  if (size < 1) return "context library SIZE " + std::to_string(size) + " is not a positive number of profiles";
  if (wlen < 1 || !(wlen & 1) || wlen > 63)
    return "context library window length " + std::to_string(wlen) +
           " is not supported: the window must be odd and 1..63 columns";
  C.K = size; C.W = wlen;
  C.bias.assign(size, 0.0);
  C.w.assign((size_t)wlen * 20 * size, 0.0);
  C.pc.assign((size_t)size * 20, 0.0);
  const int center = (wlen - 1) / 2;
  for (int k = 0; k < size; ++k) {
    const std::string at = "profile " + std::to_string(k);
    do { if (!in.next(ln)) return "context library has fewer profiles than SIZE says"; } while (text_blank(ln));
    if (ln.compare(0, 14, "ContextProfile") != 0) return at + " does not start with 'ContextProfile'";
    if (!in.next(ln)) return at + " is truncated";
    if (ln.find("NAME") != std::string::npos) { if (!in.next(ln)) return at + " is truncated"; }
    if (ln.find("PRIOR") == std::string::npos) return "unable to parse 'PRIOR' of " + at;
    const double prior = atof(ln.c_str() + 5);              // ReadDouble
    if (!in.next(ln)) return at + " is truncated";
    if (ln.find("COLOR") != std::string::npos) { if (!in.next(ln)) return at + " is truncated"; }
    if (ln.find("ISLOG") == std::string::npos) return "unable to parse 'ISLOG' of " + at;
    bool is_log;                                            // ReadBool
    const char* b = ln.c_str() + 5;
    if (strchr(b, 'T') || strchr(b, '1')) is_log = true;
    else if (strchr(b, 'F') || strchr(b, '0')) is_log = false;
    else return "unable to parse 'ISLOG' of " + at;
    int plen = 0, nalph = 0;
    if (!in.next(ln) || !text_read_int(ln, "LENG", &plen)) return "unable to parse 'LENG' of " + at;
    if (plen != wlen)
      return at + " has window length " + std::to_string(plen) + ", the library " + std::to_string(wlen);
    if (!in.next(ln) || !text_read_int(ln, "ALPH", &nalph)) return "unable to parse 'ALPH' of " + at;
    if (nalph != 20) return "alphabet size of " + at + " is " + std::to_string(nalph) + ", not 20";
    C.bias[k] = log(prior);                                 // Read (ISLOG T) or TransformToLog (ISLOG F): the same log
    if (std::isnan(C.bias[k]) || C.bias[k] == HUGE_VAL) return "PRIOR of " + at + " is not a probability";
    if (!in.next(ln)) return at + " is truncated";          // alphabet description line
    uint64_t seen = 0;
    int nrows = 0, row = -1;
    // the reference's loop condition, `buffer[0] != '/' && buffer[1] != '/'`
    while (in.next(ln) && !(ln.size() >= 1 && ln[0] == '/') && !(ln.size() >= 2 && ln[1] == '/')) {
      const char* q = ln.c_str();
      if (!text_strtoi(q, &row)) return "a row of " + at + " has no column number";
      row -= 1;
      const std::string col = at + ", column " + std::to_string(row + 1);
      if (row < 0 || row >= wlen) return col + " lies outside the window";
      if (seen >> row & 1) return col + " is given twice";
      seen |= uint64_t(1) << row;
      ++nrows;
      for (int a = 0; a < 20; ++a) {
        bool ok = true;
        const int v = text_strastoi(q, ok);
        if (!ok) return col + " has fewer than 20 values";
        const double lin = pow(2, -static_cast<double>(v) / 1000);     // kScale
        const double lg = log(lin);
        if (!std::isfinite(lg))
          return col + ", amino acid " + std::to_string(a) + ": 2^(-" + std::to_string(v) +
                 "/1000) is not a positive finite probability ('*' reads as 2147483647)";
        C.w[((size_t)row * 20 + a) * size + k] = lg;
        if (row == center) C.pc[(size_t)k * 20 + a] = is_log ? exp(lg) : lin;
      }
    }
    if (nrows != wlen || row != wlen - 1)
      return at + " should have " + std::to_string(wlen) + " columns, the last numbered " + std::to_string(wlen) +
             ", but has " + std::to_string(nrows) + ", the last numbered " + std::to_string(row + 1);
  }
  C.ww.assign(wlen, 0.0);
  C.ww[center] = wcenter;
  for (int d = 1; d <= center; ++d) C.ww[center - d] = C.ww[center + d] = wcenter * pow(wdecay, d);
  return "";
}

#if defined(__CUDACC__) || defined(HHG_EMUL)
// score[i*K + k] = bias[k] + context score of state k at column i, over the columns beg..end-1 of the window that
// exist; counts[L][20].
//   CRF (kLibrary false): ContextScore (src/cs/crf_state-inl.h:177-189), amino acids 0..19 of all those columns in one
//     ordered double sum; ww is not read.
//   Context library (kLibrary true): cs::Emission on a count profile (src/cs/emission.h:87-103), one ordered sum over
//     the amino acids per column, each weighted by the window weight ww[j] and added in column order.
// One block of 256 threads per (256 states, column); k_crf_scores and k_lib_scores are its two instantiations.
template <bool kLibrary>
__device__ __forceinline__ void context_scores(int L, int K, int W, const double* __restrict__ w,
                                               const double* __restrict__ bias, const double* __restrict__ ww,
                                               const double* __restrict__ counts, double* __restrict__ score) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  __shared__ double s_c[64 * 20];
  __shared__ double s_ww[kLibrary ? 64 : 1];
  const int center = (W - 1) / 2;
  const int beg = max(0, i - center), end = min(L, i + center + 1);
  for (int t = threadIdx.x; t < (end - beg) * 20; t += blockDim.x) s_c[t] = counts[(size_t)beg * 20 + t];
  if (kLibrary)
    for (int t = threadIdx.x; t < W; t += blockDim.x) s_ww[t] = ww[t];
  __syncthreads();
  if (k >= K) return;
  double sc = 0.0;
  for (int c = beg, j = beg - i + center; c < end; ++c, ++j) {
    const double* wj = w + (size_t)j * 20 * K + k;
    const double* cc = s_c + (c - beg) * 20;
    if (kLibrary) {
      double s = 0.0;
#pragma unroll
      for (int a = 0; a < 20; ++a) s = __dadd_rn(s, __dmul_rn(cc[a], wj[(size_t)a * K]));
      sc = __dadd_rn(sc, __dmul_rn(s_ww[j], s));
    } else {
#pragma unroll
      for (int a = 0; a < 20; ++a) sc = __dadd_rn(sc, __dmul_rn(wj[(size_t)a * K], cc[a]));
    }
  }
  score[(size_t)i * K + k] = __dadd_rn(bias[k], sc);
}

__global__ void __launch_bounds__(256)
k_crf_scores(int L, int K, int W, const double* __restrict__ w, const double* __restrict__ bias,
             const double* __restrict__ counts, double* __restrict__ score) {
  context_scores<false>(L, K, W, w, bias, nullptr, counts, score);
}

__global__ void __launch_bounds__(256)
k_lib_scores(int L, int K, int W, const double* __restrict__ w, const double* __restrict__ bias,
             const double* __restrict__ ww, const double* __restrict__ counts, double* __restrict__ score) {
  context_scores<true>(L, K, W, w, bias, ww, counts, score);
}
#endif

// The host tail for column i: log-sum-exp over the states, emission pseudocounts, Normalize, admixture with the
// observed counts, final Normalize (crf_pseudocounts-inl.h:93-108, library_pseudocounts-inl.h:58-81,
// pseudocounts-inl.h:55-73).
//   mx0: where the maximum of the log-sum-exp starts, -DBL_MAX for a CRF, -FLT_MAX for a context library
//   (context_library-inl.h:100); ppi[K]: scores of this column (overwritten), pcs: CrfHost::pc, cnt[20]: counts of the
//   column, neff its Neff, admix: 0 constant, 1 CS-BLAST, 2 HHsearch (src/cs/pseudocounts.h:52-115)
inline void crf_column_tail(int K, double mx0, double* ppi, const double* pcs, const double* cnt, double neff, int admix,
                            double pca, double pcb, double pcc, float* out20) {
  double mx = mx0;
  for (int k = 0; k < K; ++k) if (ppi[k] > mx) mx = ppi[k];
  double sum = 0.0;
  for (int k = 0; k < K; ++k) sum += exp(ppi[k] - mx);
  const double tmp = mx + log(sum);
  double pc[20];
  for (int a = 0; a < 20; ++a) pc[a] = 0.0;
  for (int k = 0; k < K; ++k) {
    const double pk = exp(ppi[k] - tmp);
    ppi[k] = pk;
    const double* s = pcs + (size_t)k * 20;
    for (int a = 0; a < 20; ++a) pc[a] += pk * s[a];
  }
  { double s = 0.0; for (int a = 0; a < 20; ++a) s += pc[a];               // Normalize(&pc[0], 20), src/cs/utils.h:282
    if (fabs(1.0 - s) > 1e-6) { const double fac = 1.0 / s; for (int a = 0; a < 20; ++a) pc[a] *= fac; } }
  double tau;
  if (admix == 0) tau = pca;
  else if (admix == 1) { const double v = pca * (pcb + 1.0) / (pcb + neff); tau = (1.0 < v) ? 1.0 : v; }   // MIN(1.0, v)
  else if (pcc == 1.0) { const double v = pca / (1.0 + neff / pcb); tau = (1.0 < v) ? 1.0 : v; }
  else { const double v = pca / (1.0 + pow(neff / pcb, pcc)); tau = (1.0 < v) ? 1.0 : v; }
  const double t = 1 - tau;
  for (int a = 0; a < 20; ++a) pc[a] = tau * pc[a] + t * cnt[a] / neff;
  { double s = 0.0; for (int a = 0; a < 20; ++a) s += pc[a];               // Normalize(p, 1.0), src/cs/profile-inl.h:175
    if (fabs(1.0 - s) > 1e-6 && s != 0.0) { const double fac = 1.0 / s; for (int a = 0; a < 20; ++a) pc[a] *= fac; } }
  for (int a = 0; a < 20; ++a) out20[a] = (float)pc[a];
}

}  // namespace hhg
