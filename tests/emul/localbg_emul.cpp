// tests/emul/localbg_emul.cpp -- TEST INFRASTRUCTURE: runs the product's local composition correction kernel
// (hh-suite_b200/csrc/hhg_localbg.cuh, unmodified source) on the CPU through tests/emul/cuda_emul.h.  Built by
// tests/test_localbg_cpu.py:
//   g++ -O1 -std=c++20 -ffp-contract=off -fPIC -shared -pthread -o tests/emul/liblocalbgemul.so tests/emul/localbg_emul.cpp
#include "cuda_emul.h"

// the IEEE operations the kernel names, as the host computes them (correctly rounded, no contraction)
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fsqrt_rn(float a) { return std::sqrt(a); }
inline double __ddiv_rn(double a, double b) { return a / b; }
inline float __double2float_rn(double a) { return (float)a; }

#include "../../hh-suite_b200/csrc/hhg_localbg.cuh"

using namespace hhg;

// k_local_bg over n segments {src, dst, L} of the record arrays src / dst (28 floats per record), on `blocks` CTAs of
// `threads` threads (a multiple of 32).
extern "C" void emul_local_bg(int n, const long long* seg3, const float* src, float* dst, const float* pb, int D,
                              int blocks, int threads) {
  std::vector<LocalBgSeg> seg(n);
  for (int k = 0; k < n; ++k) seg[k] = LocalBgSeg{seg3[3 * k], seg3[3 * k + 1], (int)seg3[3 * k + 2], 0};
  emul_launch(emul_dim3((unsigned)blocks), (unsigned)threads, k_local_bg, n, (const LocalBgSeg*)seg.data(), src, dst,
              pb, D);
}
