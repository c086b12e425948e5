// hh-suite_b200/csrc/hhg_topk.cuh -- on-device top-K selection of a plan's hit records, the step between the
// Viterbi stage of one GPU and the hit-list merge across GPUs (SURVEY 8e).
//
// Reference semantics kept: every aligned target yields one Hit and the merged list is ordered like a
// single-process search (/root/reference/src/hhblits.cpp:890-905 sorts the whole list; ties are broken
// deterministically here by ascending global target id).  The ordering key is a 64-bit composite
//     key = (~orderable(score) << 32) | global_id        (ascending key = descending score, ascending id)
// and is unique per target, so "the K smallest keys" is a well-defined set: an 8-pass MSD radix SELECT
// (histogram of one byte of the keys that match the prefix found so far, then a one-block scan that fixes the
// next byte of the K-th key) finds the K-th key exactly, and one compaction pass emits the K records.
// n keys are read 9 times (n <= a few million, 8 B each): microseconds next to the DP.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "hhg_kernels.cuh"

namespace hhg {

struct __align__(8) TopkRec {     // = hhg_topk_rec of include/hhg.h (56 B)
  int32_t target;                 // global target id (-1: padding)
  int32_t owner;                  // rank that aligned it
  HitRec hit;                     // 40 B
  unsigned long long key;         // composite ordering key (ascending = better)
};
static_assert(sizeof(TopkRec) == 56, "TopkRec layout");

struct TopkState {
  unsigned long long prefix;      // high bytes of the K-th smallest key fixed so far
  unsigned int krem;              // rank of the K-th key among the keys matching the prefix (1-based)
  unsigned int out_count;
  unsigned int hist[256];
};

__device__ __forceinline__ uint32_t orderable_f32(float f) {   // monotone increasing float -> uint32
  const uint32_t u = __float_as_uint(f);
  return u ^ ((u >> 31) ? 0xFFFFFFFFu : 0x80000000u);
}

// user_key != NULL: caller-supplied ranking value per request, ASCENDING = better (e.g. the reference's score_aass).
// The host has checked that every global id lies in [0, INT32_MAX] and that no caller key is NaN.
__global__ void __launch_bounds__(256)
k_topk_keys(int n, const HitRec* __restrict__ hits, int by_hit_score, int id_base, const int* __restrict__ gids,
            const float* __restrict__ user_key, unsigned long long* __restrict__ keys) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t gid = (uint32_t)(gids ? gids[k] : id_base + k);
  float v = user_key ? user_key[k] : (by_hit_score ? hits[k].hit_score : hits[k].score);
  if (v == 0.0f) v = 0.0f;      // -0.0 and +0.0 are one value: the global id breaks their tie like any other
  const uint32_t o = orderable_f32(v);
  keys[k] = ((unsigned long long)(user_key ? o : ~o) << 32) | gid;
}

// pass p (7 = most significant byte first): histogram byte p of the keys whose bytes above p equal the prefix
__global__ void __launch_bounds__(256)
k_topk_hist(int n, const unsigned long long* __restrict__ keys, int p, TopkState* st) {
  __shared__ unsigned int sh[256];
  sh[threadIdx.x] = 0;
  __syncthreads();
  const unsigned long long prefix = st->prefix;
  const int hs = (p + 1) * 8;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const unsigned long long key = keys[k];
    const bool match = (p == 7) || ((key >> hs) == prefix);
    if (match) atomicAdd(&sh[(unsigned)(key >> (p * 8)) & 255u], 1u);
  }
  __syncthreads();
  if (sh[threadIdx.x]) atomicAdd(&st->hist[threadIdx.x], sh[threadIdx.x]);
}

// one block: pick the byte value whose bucket holds the krem-th key, extend the prefix, clear the histogram
__global__ void k_topk_scan(TopkState* st) {
  if (threadIdx.x == 0) {
    unsigned int krem = st->krem, cum = 0;
    int d = 0;
    for (; d < 255; ++d) {
      const unsigned int c = st->hist[d];
      if (cum + c >= krem) break;
      cum += c;
    }
    st->prefix = (st->prefix << 8) | (unsigned long long)d;
    st->krem = krem - cum;
  }
  __syncthreads();
  st->hist[threadIdx.x] = 0;
}

// emit the records whose key is <= the K-th key: exactly K of them when keys are unique; the host reads out_count back
// and refuses the call when two requests share a global id and their tie makes it larger
__global__ void __launch_bounds__(256)
k_topk_emit(int n, const unsigned long long* __restrict__ keys, const HitRec* __restrict__ hits, int owner,
            TopkState* st, TopkRec* __restrict__ out, int cap) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const unsigned long long key = keys[k];
  if (key <= st->prefix) {
    const unsigned int pos = atomicAdd(&st->out_count, 1u);
    if (pos < (unsigned)cap) {
      TopkRec r;
      r.target = (int32_t)(uint32_t)(key & 0xFFFFFFFFull);
      r.owner = owner;
      r.hit = hits[k];
      r.key = key;
      out[pos] = r;
    }
  }
}

// fill the unused tail of a rank's K-record block with padding (target -1, worst key)
__global__ void k_topk_pad(TopkRec* out, int from, int to) {
  const int k = from + blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= to) return;
  TopkRec r{};
  r.target = -1;
  r.owner = -1;
  r.key = ~0ull;
  out[k] = r;
}

// Path rows of the merged list: row r belongs to exactly one rank; the owner copies the state string of its
// alignment (nsteps bytes) into row r of a zeroed [rows x width] byte matrix.  A byte-wise sum over the ranks
// (one ncclAllReduce) is then a gather.
__global__ void k_topk_paths(int rows, const TopkRec* __restrict__ merged, int my_rank,
                             const uint8_t* __restrict__ paths, int width, uint8_t* __restrict__ out) {
  const int r = blockIdx.x;
  if (r >= rows || merged[r].owner != my_rank) return;
  const int len = min(merged[r].hit.nsteps, width);
  const uint8_t* src = paths + merged[r].hit.path_off;   // HitRec.path_off = offset in the owner's path buffer
  for (int b = threadIdx.x; b < len; b += blockDim.x) out[(size_t)r * width + b] = src[b];
}

}  // namespace hhg
