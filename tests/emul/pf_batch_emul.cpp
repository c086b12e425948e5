// tests/emul/pf_batch_emul.cpp -- TEST INFRASTRUCTURE: runs the product's ungapped query-batch prefilter kernel and its
// host-side plan (hh-suite_b200/csrc/hhg_prefilter.cuh, unmodified source) on the CPU through tests/emul/cuda_emul_mw.h.
// Built by tests/test_pf_batch_emul_cpu.py:
//   g++ -O1 -std=c++20 -fPIC -shared -pthread -o tests/emul/libpfbatchemul.so tests/emul/pf_batch_emul.cpp
#include "cuda_emul_mw.h"

// The kernel's only shared memory is its dynamic buffer; one block is alive at a time, so a global array stands in for
// it (cuda_emul_mw.h makes __shared__ variables statics, which an extern declaration cannot be).
#undef __shared__
#define __shared__

// The SIMD and warp intrinsics the prefilter kernels use, with the semantics of the CUDA documentation.
inline unsigned atomicAdd(unsigned* p, unsigned v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
template <typename T> inline T __shfl_up_sync(unsigned, T v, unsigned d) {
  const int lane = (int)(threadIdx.x & 31), src = lane - (int)d;
  return emul_shfl(v, src < 0 ? lane : src);
}
template <typename T> inline T __shfl_down_sync(unsigned, T v, unsigned d) {
  const int lane = (int)(threadIdx.x & 31), src = lane + (int)d;
  return emul_shfl(v, src > 31 ? lane : src);
}
inline unsigned __ballot_sync(unsigned, bool pred) {
  g_emul_block->xchg[threadIdx.x] = pred ? 1 : 0;
  emul_syncwarp();
  unsigned m = 0;
  for (unsigned l = 0; l < 32; ++l) {
    const unsigned t = (threadIdx.x & ~31u) | l;
    if (t < g_emul_block->xchg.size() && g_emul_block->xchg[t]) m |= 1u << l;
  }
  emul_syncwarp();
  return m;
}
inline bool __all_sync(unsigned mask, bool pred) { return __ballot_sync(mask, pred) == mask; }
// byte i of the result = byte (selector nibble i & 7) of the 8-byte value {y, x}
inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) {
  const uint64_t v = ((uint64_t)y << 32) | x;
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xFFu) << (8 * i);
  return r;
}
inline int emul_s16(uint32_t v, int h) { return (int)(int16_t)(uint16_t)(v >> (16 * h)); }
inline uint32_t emul_pack_s16(int lo, int hi) { return (uint32_t)(uint16_t)(int16_t)lo | ((uint32_t)(uint16_t)(int16_t)hi << 16); }
// per halfword: max(min(a + b, c), 0)
inline uint32_t __viaddmin_s16x2_relu(uint32_t a, uint32_t b, uint32_t c) {
  int r[2];
  for (int h = 0; h < 2; ++h) r[h] = std::max(std::min(emul_s16(a, h) + emul_s16(b, h), emul_s16(c, h)), 0);
  return emul_pack_s16(r[0], r[1]);
}
// per halfword: max(a, b, c)
inline uint32_t __vimax3_s16x2(uint32_t a, uint32_t b, uint32_t c) {
  int r[2];
  for (int h = 0; h < 2; ++h) r[h] = std::max(std::max(emul_s16(a, h), emul_s16(b, h)), emul_s16(c, h));
  return emul_pack_s16(r[0], r[1]);
}
struct int4 { int x, y, z, w; };

namespace hhg {
alignas(128) unsigned char pf_smem[256 * 1024];
}

#include "../../hh-suite_b200/csrc/hhg_prefilter.cuh"

using namespace hhg;

// The steps of hhg_prefilter_ungapped_batch_run with host memory: plan (budget: memory-wave budget in bytes), pack,
// one emulated launch of `grid` blocks of `threads` threads per tile round.  scores: [nq][n].  *n_launch: launches,
// *n_waves: memory waves, *n_slabs: slabs of the plan.  Returns 0.
extern "C" int emul_pf_ungapped_batch(int nq, const int32_t* Lq, const uint8_t* const* prof, int offset, int n,
                                      const int32_t* L, const long long* off, const uint8_t* seq, double budget,
                                      int grid, int threads, int* scores, int* n_launch, int* n_waves, int* n_slabs) {
  long long total = 0;
  for (int k = 0; k < n; ++k) total = std::max(total, off[k] + L[k]);
  const PfBatchPlan plan = pf_plan_batch(nq, Lq, total, budget);
  std::vector<uint32_t> words(plan.slabs.size() * (size_t)kPfSlabWords);
  for (size_t s = 0; s < plan.slabs.size(); ++s) pf_pack_slab(plan, (int)s, Lq, prof, offset, words.data() + s * kPfSlabWords);
  std::vector<uint8_t> edge[2];
  for (auto& e : edge) e.assign((size_t)std::max(plan.max_slots, 1) * std::max(total, 1LL), 0xA5);
  for (const PfLaunch& la : plan.launches) {
    unsigned counter = 0;
    PfBatchParams P{};
    P.n = n; P.L = L; P.off = off; P.seq = seq;
    P.prof32 = words.data() + (size_t)la.slab0 * kPfSlabWords;
    P.slabs = plan.slabs.data() + la.slab0;
    P.nslab = la.nslab;
    P.chunk = pf_chunk(n, la.nslab, grid);
    P.nchunk = (n + P.chunk - 1) / P.chunk;
    P.offset = offset;
    P.total = total;
    P.edge_in = edge[(la.round + 1) & 1].data();
    P.edge_out = edge[la.round & 1].data();
    P.scores = scores;
    P.counter = &counter;
    emul_launch((unsigned)grid, (unsigned)threads, k_pf_ungapped_batch, P);
  }
  *n_launch = (int)plan.launches.size();
  *n_waves = plan.waves;
  *n_slabs = (int)plan.slabs.size();
  return 0;
}
