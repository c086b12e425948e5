// hh-suite_b200/csrc/hhg_prefilter.cuh -- query-batch kernels of the cs219 prefilter (Prefilter::prefilter_db,
// src/hhprefilter.cpp:430-606) and the parts they share with the single-query kernels of hhg_kernels.cuh.
// Kept apart from hhg_kernels.cuh (whose Viterbi kernels carry inline PTX) so that the CPU emulation under
// tests/emul can compile the ungapped batch kernel unchanged.
#pragma once
#include <algorithm>
#include <climits>
#include <cstdint>
#include <vector>

#include "hhg_math.cuh"

namespace hhg {

// ---------------------------------------------------------------------------------------------
// Ungapped stage for a batch of queries (the recurrence of k_prefilter_ungapped):
//   S(i,j) = max(0, min(255, S(i-1,j-1) + prof[x_j][i]) - offset);  score = max over all cells.
// Query positions are packed into SLABS of 512 positions: 32 lanes x 8 s16x2 registers, lane l owns slab positions
// [l*16, l*16+16) with the pairing of k_prefilter_ungapped at WB = 8 (register w = positions l*16+w | l*16+8+w).
// A query of at most 512 positions takes ceil(Lq/16) consecutive lanes of a slab (a SEGMENT) and shares the slab
// with other short queries; the diagonal carry into the first lane of a segment is 0, and the maximum is reduced per
// segment.  A longer query takes one full slab per 512-position tile, one tile per launch ("tile round"), and hands
// S(last position of the tile, column) to the next round through its own edge bytes, as k_prefilter_ungapped does.
// Positions past the end of a query carry p = 0: their S never exceeds their diagonal predecessor's.
// Work items are (slab, chunk of sequences) in slab-major order; a CTA takes one item at a time, reloads the slab's
// profile into shared memory only when the slab changes, and its warps take the chunk's sequences one by one.
// ---------------------------------------------------------------------------------------------
constexpr int kPfSlabWB = 8;                                      // registers per lane
constexpr int kPfSlabPos = 64 * kPfSlabWB;                        // query positions per slab
constexpr int kPfSlabWords = 220 * kPfSlabWB * 32;                // profile words per slab
constexpr int kPfBatchSmem = kPfSlabWords * 4 + 16;               // + the CTA's work-item slots
constexpr int kPfBatchScoreBytes = 8;                             // raw + corrected score per query and sequence

struct PfSlab {
  int tile;          // 0, or the tile (round) index of a query longer than one slab
  int last;          // 1: no further tile of the slab's query follows (no edge bytes written)
  int edge;          // edge slot of a query longer than one slab, -1 for slabs of short queries
  int lane_q[32];    // score row (query of the batch) of each lane, -1 = unused lane
};

struct PfBatchParams {
  int n;                      // sequences of the shard
  const int* L;
  const long long* off;
  const uint8_t* seq;
  const uint32_t* prof32;     // [nslab][220][8][32] words (p - offset | p - offset) as s16x2
  const PfSlab* slabs;        // [nslab]
  int nslab;
  int chunk, nchunk;          // sequences per work item, work items per slab
  int offset;
  long long total;            // bytes of one edge slot (sum of the shard's sequence lengths)
  const uint8_t* edge_in;     // [slot][total]: S(last position of the previous tile, column)
  uint8_t* edge_out;          // [slot][total]: written when the slab is not its query's last tile
  int* scores;                // [nq][n] running maximum over the tile rounds
  unsigned int* counter;      // work-item counter of this launch
};

__global__ void __launch_bounds__(512) k_pf_ungapped_batch(const PfBatchParams P) {
  extern __shared__ __align__(128) unsigned char pf_smem[];
  uint32_t* sprof = reinterpret_cast<uint32_t*>(pf_smem);                       // [220][8][32]
  int* s_item = reinterpret_cast<int*>(pf_smem + (size_t)kPfSlabWords * 4);     // work item of the CTA
  unsigned* s_next = reinterpret_cast<unsigned*>(s_item + 1);                    // next sequence of the item
  const int lane = threadIdx.x & 31;
  const uint32_t cap = (uint32_t)(255 - P.offset) * 0x00010001u;
  const int nitems = P.nslab * P.nchunk;
  int cur = -1;
  for (;;) {
    if (threadIdx.x == 0) { *s_item = (int)atomicAdd(P.counter, 1u); *s_next = 0u; }
    __syncthreads();
    const int item = *s_item;
    if (item >= nitems) break;
    const int slab = item / P.nchunk;
    if (slab != cur) {
      const uint32_t* src = P.prof32 + (size_t)slab * kPfSlabWords;
      for (int idx = threadIdx.x; idx < kPfSlabWords; idx += blockDim.x) sprof[idx] = src[idx];
      cur = slab;
    }
    __syncthreads();
    const PfSlab& sl = P.slabs[slab];
    const int q = sl.lane_q[lane];
    const bool seg_first = lane == 0 || sl.lane_q[lane - 1] != q;
    int seg_end = lane;
    while (seg_end < 31 && sl.lane_q[seg_end + 1] == q) ++seg_end;
    const bool first_tile = sl.tile == 0;
    const uint8_t* edge_in = first_tile ? nullptr : P.edge_in + (size_t)sl.edge * P.total;
    uint8_t* edge_out = sl.last ? nullptr : P.edge_out + (size_t)sl.edge * P.total;
    const int s0 = (item - slab * P.nchunk) * P.chunk;
    const int cnt_item = min(P.chunk, P.n - s0);
    for (;;) {
      int k = 0;
      if (lane == 0) k = (int)atomicAdd(s_next, 1u);
      k = __shfl_sync(0xffffffffu, k, 0);
      if (k >= cnt_item) break;
      const int n = s0 + k;
      const long long o = P.off[n];
      const uint8_t* x = P.seq + o;
      const int L = P.L[n];
      uint32_t S[kPfSlabWB];
#pragma unroll
      for (int w = 0; w < kPfSlabWB; ++w) S[w] = 0;
      uint32_t smax = 0;
      for (int j0 = 0; j0 < L; j0 += 32) {
        const int xl = (j0 + lane < L) ? (int)x[j0 + lane] : 0;
        int el = 0;
        if (edge_in && j0 + lane >= 1 && j0 + lane <= L) el = (int)edge_in[o + j0 + lane - 1];
        const int cnt = min(32, L - j0);
        uint32_t eout = 0;
        for (int jj = 0; jj < cnt; ++jj) {
          const int xs = __shfl_sync(0xffffffffu, xl, jj);
          const uint32_t* prow = sprof + (size_t)xs * (kPfSlabWB * 32) + lane;
          uint32_t up = __shfl_up_sync(0xffffffffu, S[kPfSlabWB - 1], 1);
          const uint32_t ein = edge_in ? (uint32_t)__shfl_sync(0xffffffffu, el, jj) : 0u;   // slab-uniform branch
          if (seg_first) up = ein << 16;          // a long query's slab is one segment: only lane 0 takes the edge
          const uint32_t carry = __byte_perm(up, S[kPfSlabWB - 1], 0x5432);
#pragma unroll
          for (int w = kPfSlabWB - 1; w >= 1; --w) S[w] = __viaddmin_s16x2_relu(S[w - 1], prow[w * 32], cap);
          S[0] = __viaddmin_s16x2_relu(carry, prow[0], cap);
#pragma unroll
          for (int w = 0; w < kPfSlabWB; w += 2) smax = __vimax3_s16x2(smax, S[w], S[w + 1]);
          if (edge_out) {
            const uint32_t e = __shfl_sync(0xffffffffu, S[kPfSlabWB - 1] >> 16, 31);
            if (lane == jj) eout = e;
          }
        }
        if (edge_out && lane < cnt) edge_out[o + j0 + lane] = (uint8_t)eout;
      }
      // segmented maximum: after the step of distance d, lane l holds the maximum over [l, min(l + 2d - 1, seg_end)]
      uint32_t m = max(smax & 0xFFFFu, smax >> 16);
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, m, d);
        if (lane + d <= seg_end) m = max(m, v);
      }
      if (seg_first && q >= 0) {
        int* dst = P.scores + (size_t)q * P.n + n;
        *dst = first_tile ? (int)m : max(*dst, (int)m);
      }
    }
    __syncthreads();
  }
}

// Host-side plan of a batch: queries of at most 512 positions are packed first-fit decreasing into slabs of 32 lanes
// x 16 positions; a longer query takes one slab per tile.  Memory waves: every long query keeps two edge slots of
// `total` bytes (ping-pong between tile rounds) while its wave runs, so the long queries (longest first) are cut into
// waves whose slots stay within `budget` bytes, at least one query per wave; the short slabs run in the first wave.
// A wave costs one launch per tile round: ceil(longest query of the wave / 512).
struct PfLaunch { int slab0, nslab, round; };

struct PfBatchPlan {
  std::vector<PfSlab> slabs;         // in launch order
  std::vector<PfLaunch> launches;
  std::vector<int> lane0;            // first lane of each short query in its slab
  int max_slots = 0;                 // edge slots of the largest wave
  int waves = 0;
};

inline PfBatchPlan pf_plan_batch(int nq, const int32_t* Lq, long long total, double budget) {
  PfBatchPlan plan;
  plan.lane0.assign(nq, 0);
  auto lanes_of = [&](int q) { return (Lq[q] + 15) / 16; };
  auto tiles_of = [&](int q) { return (Lq[q] + kPfSlabPos - 1) / kPfSlabPos; };
  std::vector<int> shorts, longs;
  for (int q = 0; q < nq; ++q) (Lq[q] <= kPfSlabPos ? shorts : longs).push_back(q);
  std::stable_sort(shorts.begin(), shorts.end(), [&](int a, int b) { return lanes_of(a) > lanes_of(b); });
  std::stable_sort(longs.begin(), longs.end(), [&](int a, int b) { return Lq[a] > Lq[b]; });
  PfSlab empty{};
  empty.tile = 0; empty.last = 1; empty.edge = -1;
  for (int l = 0; l < 32; ++l) empty.lane_q[l] = -1;
  std::vector<PfSlab> short_slabs;
  std::vector<int> used;                            // lanes taken in each short slab
  for (int q : shorts) {
    size_t s = 0;
    while (s < used.size() && used[s] + lanes_of(q) > 32) ++s;
    if (s == used.size()) { short_slabs.push_back(empty); used.push_back(0); }
    plan.lane0[q] = used[s];
    for (int l = 0; l < lanes_of(q); ++l) short_slabs[s].lane_q[used[s] + l] = q;
    used[s] += lanes_of(q);
  }
  std::vector<std::vector<int>> waves(1);
  for (int q : longs) {
    if (!waves.back().empty() && (double)(waves.back().size() + 1) * 2.0 * (double)total > budget) waves.emplace_back();
    waves.back().push_back(q);
  }
  plan.waves = (int)waves.size();
  for (size_t w = 0; w < waves.size(); ++w) {
    int rounds = 1;
    for (int q : waves[w]) rounds = std::max(rounds, tiles_of(q));
    plan.max_slots = std::max(plan.max_slots, (int)waves[w].size());
    for (int t = 0; t < rounds; ++t) {
      const int slab0 = (int)plan.slabs.size();
      if (w == 0 && t == 0) plan.slabs.insert(plan.slabs.end(), short_slabs.begin(), short_slabs.end());
      for (size_t slot = 0; slot < waves[w].size(); ++slot) {
        const int q = waves[w][slot];
        if (t >= tiles_of(q)) continue;
        PfSlab sl{};
        sl.tile = t; sl.last = (t == tiles_of(q) - 1); sl.edge = (int)slot;
        for (int l = 0; l < 32; ++l) sl.lane_q[l] = q;
        plan.slabs.push_back(sl);
      }
      if ((int)plan.slabs.size() > slab0) plan.launches.push_back({slab0, (int)plan.slabs.size() - slab0, t});
    }
  }
  return plan;
}

// Profile words of slab s (kPfSlabWords): lane l of a segment that starts at lane l0 covers query positions
// tile*512 + (l - l0)*16 .. +16; word w = (position base+w | position base+8+w), each as the s16 value p - offset.
inline void pf_pack_slab(const PfBatchPlan& plan, int s, const int32_t* Lq, const uint8_t* const* prof, int offset,
                         uint32_t* out) {
  const PfSlab& sl = plan.slabs[s];
  const uint32_t pad = (uint32_t)(uint16_t)(int16_t)(-offset);
  for (int l = 0; l < 32; ++l) {
    const int q = sl.lane_q[l];
    const int base = q < 0 ? 0 : sl.tile * kPfSlabPos + (l - (Lq[q] <= kPfSlabPos ? plan.lane0[q] : 0)) * 16;
    for (int k = 0; k < 220; ++k)
      for (int w = 0; w < kPfSlabWB; ++w) {
        uint32_t v = pad | (pad << 16);
        if (q >= 0) {
          const int plo = base + w, phi = base + kPfSlabWB + w;
          const uint8_t* pr = prof[q] + (size_t)k * Lq[q];
          const uint32_t lo = plo < Lq[q] ? (uint32_t)(uint16_t)(int16_t)((int)pr[plo] - offset) : pad;
          const uint32_t hi = phi < Lq[q] ? (uint32_t)(uint16_t)(int16_t)((int)pr[phi] - offset) : pad;
          v = lo | (hi << 16);
        }
        out[((size_t)k * kPfSlabWB + w) * 32 + l] = v;
      }
  }
}

// Work-item size of a launch over nslab slabs: about four items per CTA, enough to balance the sequences' lengths and
// few enough to keep the profile reloads rare.
inline int pf_chunk(int n, int nslab, long long ctas) {
  return (int)std::max(32LL, std::min(4096LL, ((long long)n * nslab + 4 * ctas - 1) / (4 * ctas)));
}

// ---------------------------------------------------------------------------------------------
// Stage-1 selection of Prefilter::prefilter_db on the device (src/hhprefilter.cpp:477-506) for nq score rows of n
// sequences (blockIdx.y = row): the raw scores never travel to the host.  Pass 1 applies the length correction (:477)
// and histograms the corrected scores per row; the host picks each row's cut from its 1024-bin histogram, which also
// gives the exact sizes of its lists A (above the cut) and B (at the cut); pass 2 compacts the survivors of every row
// into its own region.
// ---------------------------------------------------------------------------------------------
constexpr int kPfHistBins = 1024;   // bin = corrected score + 512, clamped
constexpr int kPfHistBias = 512;

__global__ void __launch_bounds__(256)
k_pf_correct_hist(int n, const int* __restrict__ L, const int* __restrict__ raw, const float* __restrict__ flog2_Lq,
                  int bit_factor, int* __restrict__ corr, unsigned int* __restrict__ hist) {
  __shared__ unsigned int sh[kPfHistBins];
  const int row = blockIdx.y;
  raw += (size_t)row * n; corr += (size_t)row * n; hist += (size_t)row * kPfHistBins;
  const float lq = flog2_Lq[row];
  for (int b = threadIdx.x; b < kPfHistBins; b += blockDim.x) sh[b] = 0;
  __syncthreads();
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const int c = raw[k] - (int)__fmul_rn((float)bit_factor, __fadd_rn(lq, flog2_dev((float)L[k])));
    corr[k] = c;
    atomicAdd(&sh[min(max(c + kPfHistBias, 0), kPfHistBins - 1)], 1u);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < kPfHistBins; b += blockDim.x)
    if (sh[b]) atomicAdd(&hist[b], sh[b]);
}

struct PfCut {
  int cut, take_eq;     // survivors: corr > cut -> list A; corr == cut && take_eq -> list B
  int a_off, b_off;     // first slot of the row's lists in ids_a / score_a and ids_b
};

// list order inside a row is restored by the caller's sort
__global__ void __launch_bounds__(256)
k_pf_compact(int n, const int* __restrict__ corr, const PfCut* __restrict__ cuts, int* __restrict__ ids_a,
             int* __restrict__ score_a, int* __restrict__ ids_b, unsigned int* __restrict__ counters) {
  const int row = blockIdx.y;
  const PfCut C = cuts[row];
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = k < n ? corr[(size_t)row * n + k] : INT_MIN;
  const bool a = k < n && c > C.cut;
  const bool b = k < n && C.take_eq && c == C.cut;
  const unsigned ma = __ballot_sync(0xffffffffu, a), mb = __ballot_sync(0xffffffffu, b);
  const int lane = threadIdx.x & 31;
  unsigned base_a = 0, base_b = 0;
  if (lane == 0) {
    if (ma) base_a = atomicAdd(&counters[2 * row], (unsigned)__popc(ma));
    if (mb) base_b = atomicAdd(&counters[2 * row + 1], (unsigned)__popc(mb));
  }
  base_a = __shfl_sync(0xffffffffu, base_a, 0);
  base_b = __shfl_sync(0xffffffffu, base_b, 0);
  const unsigned below = (1u << lane) - 1u;
  if (a) { const unsigned pos = C.a_off + base_a + __popc(ma & below); ids_a[pos] = k; score_a[pos] = c; }
  if (b) ids_b[C.b_off + base_b + __popc(mb & below)] = k;
}

// ---------------------------------------------------------------------------------------------
// Gapped byte Smith-Waterman of prefilter stage 2 (Prefilter::swStripedByte, src/hhprefilter.cpp:70-212) for one
// sequence, by one warp: the 32 lanes are the 32 byte lanes of the reference's AVX2 vector (lane k owns query positions
// k*W + j), the full-width byte shift is __shfl_up, the movemask test is __all_sync, and the lazy-F loop does not update
// E, as in the reference (its score can depend on the striping, SURVEY App. D-5).  sprof: striped profile
// [220][W][32], byte (k, j, lane) = position lane*W + j (bias pad).  Hst / Hld / E: the warp's working columns,
// already offset by the lane (element j at [j*32]).  Returns the score, in every lane.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int pf_sw_sequence(const uint8_t* sprof, int W, const uint8_t* x, int L, uint8_t* Hst,
                                              uint8_t* Hld, uint8_t* E, int go, int ge, int bias, int lane) {
  for (int j = 0; j < W; ++j) { Hst[j * 32] = 0; Hld[j * 32] = 0; E[j * 32] = 0; }
  int vmax = 0;
  for (int i = 0; i < L; ++i) {
    int vF = 0, vMaxCol = 0;
    int vH = __shfl_up_sync(0xffffffffu, (int)Hst[(W - 1) * 32], 1);
    if (lane == 0) vH = 0;
    const uint8_t* row = sprof + (size_t)x[i] * W * 32 + lane;
    { uint8_t* t = Hld; Hld = Hst; Hst = t; }
    for (int j = 0; j < W; ++j) {
      int h = min(vH + (int)row[j * 32], 255);
      h = max(h - bias, 0);
      int e = E[j * 32];
      h = max(h, e);
      h = max(h, vF);
      vMaxCol = max(vMaxCol, h);
      Hst[j * 32] = (uint8_t)h;
      h = max(h - go, 0);
      e = max(max(e - ge, 0), h);
      E[j * 32] = (uint8_t)e;
      vF = max(max(vF - ge, 0), h);
      vH = Hld[j * 32];
    }
    // lazy F (:158-196)
    int j = 0;
    vF = __shfl_up_sync(0xffffffffu, vF, 1);
    if (lane == 0) vF = 0;
    for (;;) {
      int h = Hst[j * 32];
      const bool done = max(vF - max(h - go, 0), 0) == 0;
      if (__all_sync(0xffffffffu, done)) break;
      h = max(h, vF);
      vMaxCol = max(vMaxCol, h);
      Hst[j * 32] = (uint8_t)h;
      vF = max(vF - ge, 0);
      if (++j >= W) {
        j = 0;
        vF = __shfl_up_sync(0xffffffffu, vF, 1);
        if (lane == 0) vF = 0;
      }
    }
    vmax = max(vmax, vMaxCol);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) vmax = max(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
  return vmax;
}

// Stage 2 for the requests of a batch of queries in one launch.  The host groups the requests by query; a work item is
// (query, chunk of its requests).  A CTA takes one item at a time and copies the query's striped profile into shared
// memory only when the query changes; a query whose profile does not fit next to its working columns is read from
// L2, exactly when k_prefilter_sw<false> would be chosen for it.
struct SwBatchQuery {
  int W;                 // stripes of the query (ceil(Lq / 32))
  int smem;              // 1: the profile is staged in shared memory (at offset 0)
  int work_off;          // shared-memory offset of the working columns (after the staged profile, if any)
  long long prof_off;    // first byte of the query's striped profile in prof
};

struct SwBatchParams {
  int nitem;
  const int4* items;             // x: query, y: first request (grouped order), z: number of requests
  const SwBatchQuery* queries;
  const int* ids;                // [n] sequence ids, grouped by query
  const int* L;
  const long long* off;
  const uint8_t* seq;
  const uint8_t* prof;           // the queries' striped profiles, concatenated
  int ctrl_off;                  // shared-memory offset of the CTA's work-item slots (after every query's working set)
  int gap_open, gap_extend, bias;
  int* scores;                   // [n] in grouped order
  unsigned int* counter;
};

__global__ void __launch_bounds__(256) k_prefilter_sw_batch(const SwBatchParams P) {
  extern __shared__ __align__(128) unsigned char pf_smem[];
  int* s_item = reinterpret_cast<int*>(pf_smem + P.ctrl_off);
  unsigned* s_next = reinterpret_cast<unsigned*>(s_item + 1);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int staged = -1;   // query whose profile is in shared memory, -1 when none is intact
  for (;;) {
    if (threadIdx.x == 0) { *s_item = (int)atomicAdd(P.counter, 1u); *s_next = 0u; }
    __syncthreads();
    const int item = *s_item;
    if (item >= P.nitem) break;
    const int4 it = P.items[item];
    const SwBatchQuery Q = P.queries[it.x];
    if (Q.smem && it.x != staged) {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(P.prof + Q.prof_off);
      uint32_t* dst = reinterpret_cast<uint32_t*>(pf_smem);
      for (int idx = threadIdx.x; idx < 220 * Q.W * 8; idx += blockDim.x) dst[idx] = src[idx];
      staged = it.x;
    } else if (!Q.smem) {
      staged = -1;     // this query's working columns start at offset 0, over the staged profile
    }
    __syncthreads();
    uint8_t* Hst = pf_smem + Q.work_off + (size_t)warp * 3 * Q.W * 32 + lane;
    for (;;) {
      int r = 0;
      if (lane == 0) r = (int)atomicAdd(s_next, 1u);
      r = __shfl_sync(0xffffffffu, r, 0);
      if (r >= it.z) break;
      const int req = it.y + r;
      const int id = P.ids[req];
      const uint8_t* x = P.seq + P.off[id];
      // two call sites, so that the staged profile is read with shared-memory loads (the branch is CTA-uniform)
      const int v = Q.smem
          ? pf_sw_sequence(pf_smem, Q.W, x, P.L[id], Hst, Hst + (size_t)Q.W * 32, Hst + (size_t)2 * Q.W * 32,
                           P.gap_open, P.gap_extend, P.bias, lane)
          : pf_sw_sequence(P.prof + Q.prof_off, Q.W, x, P.L[id], Hst, Hst + (size_t)Q.W * 32,
                           Hst + (size_t)2 * Q.W * 32, P.gap_open, P.gap_extend, P.bias, lane);
      if (lane == 0) P.scores[req] = v;
      __syncwarp();
    }
    __syncthreads();
  }
}

}  // namespace hhg
