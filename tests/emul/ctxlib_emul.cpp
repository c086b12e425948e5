// tests/emul/ctxlib_emul.cpp -- TEST INFRASTRUCTURE: runs the product's context-library score kernel k_lib_scores
// (hh-suite_b200/csrc/hhg_crf.cuh, unmodified source) on the CPU through tests/emul/cuda_emul_mw.h.
// Built by tests/test_ctxlib_cpu.py into a temporary directory:
//   g++ -O1 -std=c++20 -ffp-contract=off -fPIC -shared -pthread -DHHG_EMUL -o libctxlibemul.so tests/emul/ctxlib_emul.cpp
#include "cuda_emul_mw.h"

#include "../../hh-suite_b200/csrc/hhg_crf.cuh"

using namespace hhg;

// w[W*20*K] log-probabilities ([window][aa][profile]), bias[K] log priors, ww[W] window weights, counts[L*20]
extern "C" void emul_lib_scores(int L, int K, int W, const double* w, const double* bias, const double* ww,
                                const double* counts, double* score) {
  emul_launch2((unsigned)((K + 255) / 256), (unsigned)L, 256, k_lib_scores, L, K, W, w, bias, ww, counts, score);
}
