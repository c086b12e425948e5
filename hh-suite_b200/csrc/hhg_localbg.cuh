// hh-suite_b200/csrc/hhg_localbg.cuh -- local amino-acid composition correction (-sc 5 / -scwin D):
// HMM::DivideBySqrtOfLocalBackgroundFreqs (src/hhhmm.cpp:1979-2035) on 112-byte column records.
//
// For every amino acid a, pnul[i][a] is 10*pb[a] plus the sum of p[.][a] over the window of 2D+1 columns around column
// i (over the whole profile when L <= 2D+1; the first and last D columns take the sum of the first / last full window),
// and p[i][a] becomes p[i][a] / sqrt(fac * pnul[i][a]) with fac = 1/(2D+11) (1/(L+10) for the short profile).  The
// window sum is a float recurrence, pnul[i] = (pnul[i-1] + p[i+D]) - p[i-1-D], so it is computed in the reference's
// order: one lane per amino acid walks the columns of one segment left to right.  Rows 0 and L+1 of the reference's
// profile are not touched there and have no record here.
//
// Self-contained (no ColRec, no float4) so that tests/emul/ can run it on the CPU through cuda_emul.h.
#pragma once

namespace hhg {

// One profile: L records starting at record src of the source array, written to record dst of the output array.
struct LocalBgSeg {
  long long src, dst;
  int L, pad;
};

constexpr int kLocalBgThreads = 256;   // 8 warps per CTA, one segment per warp at a time
constexpr int kLocalBgUnroll = 8;      // columns whose loads are issued before their share of the add chain
constexpr int kRecFloats = 28;         // floats per 112-byte record: p[20], 7 transitions, ss

// p / sqrt(fac * s), single precision throughout like the reference (vmulss, vsqrtss, vdivss)
__device__ __forceinline__ float local_bg_div(float p, float fac, float s) {
  return __fdiv_rn(p, __fsqrt_rn(__fmul_rn(fac, s)));
}

// Columns lo..hi (1-based) of amino acid a divided with one window sum s.
__device__ __forceinline__ void local_bg_const(const float* __restrict__ s0, float* __restrict__ d0, int a, int lo,
                                               int hi, float fac, float s) {
  constexpr int U = kLocalBgUnroll;
  const float den = __fsqrt_rn(__fmul_rn(fac, s));
  for (int i = lo; i <= hi; i += U) {
    float v[U];
#pragma unroll
    for (int k = 0; k < U; ++k)
      if (i + k <= hi) v[k] = s0[(size_t)(i + k - 1) * kRecFloats + a];
#pragma unroll
    for (int k = 0; k < U; ++k)
      if (i + k <= hi) d0[(size_t)(i + k - 1) * kRecFloats + a] = __fdiv_rn(v[k], den);
  }
}

// nseg segments, grid-striding one warp per segment.  src and dst must not overlap: the recurrence reads raw columns
// D+1 behind the column it writes.  Lanes 0..19 own one amino acid each; all 32 lanes copy the transitions and ss.
__global__ void __launch_bounds__(kLocalBgThreads)
k_local_bg(int nseg, const LocalBgSeg* __restrict__ seg, const float* __restrict__ src, float* __restrict__ dst,
           const float* __restrict__ pb, int D) {
  constexpr int U = kLocalBgUnroll;
  const int lane = threadIdx.x & 31;
  const int warp = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), nwarps = (int)((gridDim.x * blockDim.x) >> 5);
  for (int g = warp; g < nseg; g += nwarps) {
    const LocalBgSeg sg = seg[g];
    const int L = sg.L;
    const float* s0 = src + (size_t)sg.src * kRecFloats;
    float* d0 = dst + (size_t)sg.dst * kRecFloats;
    for (int e = lane; e < L * 8; e += 32) {
      const size_t off = (size_t)(e >> 3) * kRecFloats + 20 + (e & 7);
      d0[off] = s0[off];
    }
    if (lane >= 20) continue;
    const int a = lane;
    // L <= 2D+1 in 64 bits: any D >= 16383 takes the whole-profile branch for every record length
    const bool whole = (long long)L <= 2LL * D + 1;
    const int W = whole ? L : 2 * D + 1;
    float s = __fmul_rn(10.0f, pb[a]);
    for (int i = 1; i <= W; i += U) {
      float v[U];
#pragma unroll
      for (int k = 0; k < U; ++k)
        if (i + k <= W) v[k] = s0[(size_t)(i + k - 1) * kRecFloats + a];
#pragma unroll
      for (int k = 0; k < U; ++k)
        if (i + k <= W) s = __fadd_rn(s, v[k]);
    }
    // fac = 1.0 / N in double, stored to float (N = L + 10 or 2D + 11, an exact integer either way)
    const float fac = __double2float_rn(__ddiv_rn(1.0, whole ? (double)(L + 10) : (double)(2LL * D + 11)));
    if (whole) {
      local_bg_const(s0, d0, a, 1, L, fac, s);
      continue;
    }
    local_bg_const(s0, d0, a, 1, D + 1, fac, s);
    const int hi = L - D;
    for (int i = D + 2; i <= hi; i += U) {
      float p[U], in[U], out[U];
#pragma unroll
      for (int k = 0; k < U; ++k)
        if (i + k <= hi) {
          p[k] = s0[(size_t)(i + k - 1) * kRecFloats + a];
          in[k] = s0[(size_t)(i + k + D - 1) * kRecFloats + a];
          out[k] = s0[(size_t)(i + k - D - 2) * kRecFloats + a];
        }
#pragma unroll
      for (int k = 0; k < U; ++k)
        if (i + k <= hi) {
          s = __fsub_rn(__fadd_rn(s, in[k]), out[k]);
          d0[(size_t)(i + k - 1) * kRecFloats + a] = local_bg_div(p[k], fac, s);
        }
    }
    local_bg_const(s0, d0, a, hi + 1, L, fac, s);
  }
}

}  // namespace hhg
