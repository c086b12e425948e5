// hhg_crf.cuh -- context-specific (CRF) pseudocounts of the query (SURVEY §8 row a12, the default branch of
// PrepareQueryHMM, src/hhfunc.cpp:143-147, and of the prefilter profile, src/hhblits.cpp): cs::CrfPseudocounts::
// AddToProfile (src/cs/crf_pseudocounts-inl.h:74-110) + Pseudocounts::AddTo / AdmixTo (src/cs/pseudocounts-inl.h:41-73).
//
// Work split: the O(L * K * 13 * 20) part -- the context score of every CRF state at every column, ordered
// double-precision sums -- runs in k_crf_scores; the log-sum-exp over the K = 4000 states needs exp() and log() with
// the bits of the host's C library (the reference calls libm; CUDA's double exp is a different approximation), so the
// O(L * K) tail runs on the host threads of the library.
#pragma once
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
  std::vector<double> bias;              // [K]
  std::vector<double> w;                 // [W][20][K]  context weights, state index fastest (coalesced in the kernel)
  std::vector<double> pc;                // [K][20]     emission pseudocounts of the states (UpdatePseudocounts)
};

// cs::Crf::Read + CrfState::Read (src/cs/crf-inl.h:56-80, crf_state-inl.h:28-76) on the text of a .crf file
inline std::string crf_parse(const char* text, int64_t len, CrfHost* out) {
  CrfHost& C = *out;
  C = CrfHost();
  const char* p = text;
  const char* end = text + len;
  auto next_line = [&](std::string& ln) {
    if (p >= end) return false;
    const char* e = (const char*)memchr(p, '\n', (size_t)(end - p));
    if (!e) e = end;
    ln.assign(p, e);
    while (!ln.empty() && (ln.back() == '\r' || ln.back() == '\0')) ln.pop_back();
    p = e < end ? e + 1 : end;
    return true;
  };
  auto blank = [](const std::string& s) { for (char c : s) if ((unsigned char)c > 32) return false; return true; };
  auto strastoi = [](const char*& q, bool& ok) -> int {       // src/cs/io.h:76-92
    const char* q0 = q;
    while (*q != '\0' && !(*q >= '0' && *q <= '9') && *q != '*') ++q;
    if (*q == '\0') { ok = false; return INT_MIN; }
    if (*q == '*') { ++q; return INT_MAX; }
    int i = (q > q0 && *(q - 1) == '-') ? -atoi(q) : atoi(q);
    while (*q >= '0' && *q <= '9') ++q;
    return i;
  };
  auto read_int = [&](const std::string& ln, const char* label, int* v) {
    const size_t at = ln.find(label);
    if (at == std::string::npos) return false;
    const char* q = ln.c_str() + strlen(label);           // like ReadInt: the value follows the label at line start
    const char* q0 = q;
    while (*q != '\0' && !(*q >= '0' && *q <= '9')) ++q;
    if (*q == '\0') return false;
    *v = (q > q0 && *(q - 1) == '-') ? -atoi(q) : atoi(q);
    return true;
  };
  std::string ln;
  do { if (!next_line(ln)) return "empty CRF text"; } while (blank(ln));
  if (ln.compare(0, 3, "CRF") != 0) return "text does not start with class id 'CRF'";
  int size = 0, wlen = 0;
  if (!next_line(ln) || !read_int(ln, "SIZE", &size)) return "unable to parse CRF 'SIZE'";
  if (!next_line(ln) || !read_int(ln, "LENG", &wlen)) return "unable to parse CRF 'LENG'";
  if (size < 1) return "CRF SIZE " + std::to_string(size) + " is not a positive number of states";
  // k_crf_scores stages the window in a 64-column shared-memory tile; the reference's reader asserts on even windows
  if (wlen < 1 || !(wlen & 1) || wlen > 63)
    return "CRF window length " + std::to_string(wlen) + " is not supported: the window must be odd and 1..63 columns";
  C.K = size; C.W = wlen;
  C.bias.assign(size, 0.0);
  C.w.assign((size_t)wlen * 20 * size, 0.0);
  C.pc.assign((size_t)size * 20, 0.0);
  for (int k = 0; k < size; ++k) {
    do { if (!next_line(ln)) return "CRF has fewer states than SIZE says"; } while (blank(ln));
    if (ln.compare(0, 8, "CrfState") != 0) return "state " + std::to_string(k) + " does not start with 'CrfState'";
    if (!next_line(ln)) return "truncated state";
    if (ln.find("NAME") != std::string::npos) { if (!next_line(ln)) return "truncated state"; }
    if (ln.find("BIAS") == std::string::npos) return "unable to parse CRF state 'BIAS'";
    C.bias[k] = atof(ln.c_str() + 4);
    int slen = 0, nalph = 0;
    if (!next_line(ln) || !read_int(ln, "LENG", &slen) || slen != wlen) return "state window length differs from the CRF's";
    if (!next_line(ln) || !read_int(ln, "ALPH", &nalph) || nalph != 20) return "alphabet size of a CRF state is not 20";
    if (!next_line(ln)) return "truncated state";        // alphabet description line
    double pcw[20];
    bool have_pc = false;
    int last_row = -1;
    while (next_line(ln) && !(ln.size() >= 2 && ln[0] == '/' && ln[1] == '/') ) {
      // the reference's loop condition is `buffer[0] != '/' && buffer[1] != '/'`; rows start with a digit or "PC"
      const char* q = ln.c_str();
      bool ok = true;
      if (!(ln.size() >= 2 && ln[0] == 'P' && ln[1] == 'C')) {
        const char* q0 = q;
        while (*q != '\0' && !(*q >= '0' && *q <= '9')) ++q;
        if (*q == '\0') return "context weight row without a column number";
        const int row = ((q > q0 && *(q - 1) == '-') ? -atoi(q) : atoi(q)) - 1;
        while (*q >= '0' && *q <= '9') ++q;
        if (row < 0 || row >= wlen) return "context weight row outside the window";
        for (int a = 0; a < 20; ++a) {
          const int v = strastoi(q, ok);
          if (!ok) return "context weight row has fewer than 20 values";
          C.w[((size_t)row * 20 + a) * size + k] = static_cast<double>(v) / 1000;      // kScale
        }
        last_row = row;
      } else {
        for (int a = 0; a < 20; ++a) {
          const int v = strastoi(q, ok);
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

#if defined(__CUDACC__) || defined(HHG_EMUL)
// score[i*K + k] = bias[k] + ContextScore(state k, count profile, column i)  (src/cs/crf_state-inl.h:177-189):
// columns beg..end-1 of the window that exist, amino acids 0..19, one ordered double sum.  counts[L][20].
__global__ void __launch_bounds__(256)
k_crf_scores(int L, int K, int W, const double* __restrict__ w, const double* __restrict__ bias,
             const double* __restrict__ counts, double* __restrict__ score) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y;
  __shared__ double s_c[64 * 20];
  const int center = (W - 1) / 2;
  const int beg = max(0, i - center), end = min(L, i + center + 1);
  for (int t = threadIdx.x; t < (end - beg) * 20; t += blockDim.x) s_c[t] = counts[(size_t)beg * 20 + t];
  __syncthreads();
  if (k >= K) return;
  double sc = 0.0;
  for (int c = beg, j = beg - i + center; c < end; ++c, ++j) {
    const double* wj = w + (size_t)j * 20 * K + k;
    const double* cc = s_c + (c - beg) * 20;
#pragma unroll
    for (int a = 0; a < 20; ++a) sc = __dadd_rn(sc, __dmul_rn(wj[(size_t)a * K], cc[a]));
  }
  score[(size_t)i * K + k] = __dadd_rn(bias[k], sc);
}
#endif

// The host tail for column i: log-sum-exp over the states, emission pseudocounts, Normalize, admixture with the
// observed counts, final Normalize (crf_pseudocounts-inl.h:93-108, pseudocounts-inl.h:55-73).
//   ppi[K]: scores of this column (overwritten), pcs: CrfHost::pc, cnt[20]: counts of the column, neff its Neff,
//   admix: 0 constant, 1 CS-BLAST, 2 HHsearch (src/cs/pseudocounts.h:52-115)
inline void crf_column_tail(int K, double* ppi, const double* pcs, const double* cnt, double neff, int admix, double pca,
                            double pcb, double pcc, float* out20) {
  double mx = -DBL_MAX;
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
