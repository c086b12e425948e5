// hh-suite_b200/csrc/hhg_kernels.cuh -- sm_90a kernels of the HH-suite hot path.
//
// Viterbi HMM-HMM forward pass (replaces Viterbi::AlignWith[Out]CellOff[AndSS],
// src/hhviterbialgorithm.cpp:29-497 of the reference) and the byte backtrace
// (Viterbi::Backtrace, src/hhviterbi.cpp:83-160).
//
// Mapping (GPU-first, not the reference's 8-lane AVX2 row sweep):
//   * one LANE = one target; one WARP-JOB = 32 length-sorted targets; the job's DP matrix is cut
//     into STRIPS of R query rows.  A work item is (job, strip); persistent warps pull items from
//     an atomic queue in (job, strip) order, so consecutive strips of a job run on different
//     warps as a skewed wavefront: strip s+1 trails strip s by a few columns and receives the
//     5-state boundary row through L2 as tagged 64-bit words (three coalesced accesses per column).
//   * inside a strip a lane sweeps target columns left to right and keeps the 5 pair-state
//     values of its R rows in registers; the R query rows (20 emissions + 7 transitions each)
//     are TMA-bulk-staged (cp.async.bulk + mbarrier) into the warp's shared-memory slice and
//     read back as warp-uniform broadcast LDS.128.
//   * target operands stream from a JOB-INTERLEAVED copy of the job's column records,
//     [column][k = 0..6][lane] float4 (built per plan by k_interleave_cols), so each of the 7 loads of a
//     column is ONE coalesced 512-byte warp request (4 L1TEX wavefronts instead of 32 when every lane
//     reads its own 112-byte record).  Lane l only ever touches the elements [k][l], so every lane cp.asyncs its own
//     7 x 16 B of column j+1 into a lane-private slot of a two-column shared-memory ring while column j computes, and
//     reads them back with its own LDS.128 after its own cp.async.wait_group: no barrier, no elected lane, no
//     cross-lane ordering, and no registers held for the next column.
//   * 1 backtrace byte per cell, packed 4 rows per 32-bit word and stored lane-interleaved so
//     every warp store writes one full 128-byte line.
// Arithmetic is the reference's, operation for operation (unfused fp32 mul/add in the same order,
// strict '>' tie rules), so scores and backtrace bytes are bit-identical to the AVX2 (no-FMA) build.
#pragma once
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#ifndef HHG_MAX3
#define HHG_MAX3 1   // MM-state maximum as a chain of maxima + equality selects (same bits as the '>' chain)
#endif

#include "hhg_math.cuh"
#include "hhg_prefilter.cuh"

namespace hhg {

constexpr int kWarpsPerCta = 4;

struct __align__(16) ColRec {      // one profile column = operands of DP cell (., j)   (112 B)
  float p[20];
  float m2m, m2d, d2m, d2d, i2m;   // tr[j-1][M2M,M2D,D2M,D2D,I2M]
  float i2i, m2i;                  // tr[j][I2I,M2I]
  uint32_t ss;                     // ss_pred*11+ss_conf of column j
};
static_assert(sizeof(ColRec) == 112, "ColRec must be 7 x 16 bytes");

// Boundary hand-off between consecutive strips of a job: the 5 pair-state values of the strip's last
// row at one column, each paired with a tag in one 64-bit word.  The PTX memory model makes every aligned
// 64-bit element of a relaxed vector access single-copy atomic, so a word whose tag names the producing
// strip of this run carries that strip's value: the consumer lane re-reads until all five tags match --
// per-lane dataflow synchronisation with no fences, flags or L1 invalidations.
// A column of a job holds the 32 lanes' slots part-interleaved, [part][lane]: words 0-1 and 2-3 as 16-byte
// parts, word 4 as an 8-byte part, so each of the three warp-wide accesses is one contiguous, coalesced run.
struct __align__(8) BndSlot {
  unsigned long long w[5];
};
static_assert(sizeof(BndSlot) == 40, "BndSlot must be five 64-bit words");

__device__ __forceinline__ unsigned long long tagged(float v, uint32_t tag) {
  return ((unsigned long long)tag << 32) | __float_as_uint(v);
}
// col: the job's 32 slots of one column
__device__ __forceinline__ void st_slot(BndSlot* col, int lane, float mm, float dg, float mi, float gd, float im,
                                        uint32_t tag) {
  unsigned long long* p = reinterpret_cast<unsigned long long*>(col);
  asm volatile("st.relaxed.gpu.global.v2.b64 [%0], {%1,%2};" ::"l"(p + 2 * lane), "l"(tagged(mm, tag)),
               "l"(tagged(dg, tag)) : "memory");
  asm volatile("st.relaxed.gpu.global.v2.b64 [%0], {%1,%2};" ::"l"(p + 64 + 2 * lane), "l"(tagged(mi, tag)),
               "l"(tagged(gd, tag)) : "memory");
  asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p + 128 + lane), "l"(tagged(im, tag)) : "memory");
}
// The five tags come back separately (the upper halves of the words) and stay live until the slot is consumed:
// a dead destination register of an in-flight load gets reused by ptxas and the re-use then stalls on the load.
__device__ __forceinline__ void ld_slot(const BndSlot* col, int lane, float& mm, float& dg, float& mi, float& gd,
                                        float& im, uint32_t (&tag)[5]) {
  const unsigned long long* p = reinterpret_cast<const unsigned long long*>(col);
  unsigned long long w0, w1, w2, w3, w4;
  asm volatile("ld.relaxed.gpu.global.v2.b64 {%0,%1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p + 2 * lane) : "memory");
  asm volatile("ld.relaxed.gpu.global.v2.b64 {%0,%1}, [%2];" : "=l"(w2), "=l"(w3) : "l"(p + 64 + 2 * lane) : "memory");
  asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w4) : "l"(p + 128 + lane) : "memory");
  mm = __uint_as_float((uint32_t)w0); tag[0] = (uint32_t)(w0 >> 32);
  dg = __uint_as_float((uint32_t)w1); tag[1] = (uint32_t)(w1 >> 32);
  mi = __uint_as_float((uint32_t)w2); tag[2] = (uint32_t)(w2 >> 32);
  gd = __uint_as_float((uint32_t)w3); tag[3] = (uint32_t)(w3 >> 32);
  im = __uint_as_float((uint32_t)w4); tag[4] = (uint32_t)(w4 >> 32);
}
// slot valid for tag t: all five words carry t
__device__ __forceinline__ bool slot_ok(const uint32_t (&tag)[5], uint32_t want) {
  return ((tag[0] ^ want) | (tag[1] ^ want) | (tag[2] ^ want) | (tag[3] ^ want) | (tag[4] ^ want)) == 0u;
}

// One 32-target warp job of a plan (plan_build): up to 32 length-sorted requests of one query, one per lane.
struct JobDesc {
  long long ss_off;   // offset (in 32-lane blocks) of the job's per-strip maxima (absolute over all waves)
  long long bt_off;   // offset (in uint32 words) into bt, relative to the job's memory wave
  long long bnd_off;  // offset (in slots) into bnd
  long long co_off;   // offset (in uint32 words) of the job's cell-off words
  long long jc_off;   // offset (in float4) of the job's operand stream
  int Lmax;           // length of the job's longest (first) target
  int query;          // index of the job's query in the query batch
  int nstrips;        // ceil(Lq / R)
  int Lq;             // length of the job's query
  int qrow0;          // first row record of the job's query in qrec
};
static_assert(sizeof(JobDesc) == 64, "JobDesc: 5 x int64 + 5 x int32, tail padding only");

// One request of a plan: one (query, target) alignment, traced by lane `lane` of job `job`.
struct ReqDesc {
  long long path_off;  // offset into the plan's path bytes and per-step scores (capacity Lq + Lt + 2)
  int job;             // absolute job index
  int lane;            // lane in the job
  int target;          // target id in the shard
  int Lt;              // target length
  int Lq;              // query length
};
static_assert(sizeof(ReqDesc) == 32, "ReqDesc: 1 x int64 + 5 x int32, tail padding only");

struct VitParams {
  // queries: a plan may hold several (query-batch mode, hhblits_omp semantics); every job belongs to one of them
  const float4* qrec;        // query row records (rows 1..Lq of every query, each block zero padded to a multiple of 48)
  const JobDesc* jobs;       // [njobs] this wave's jobs (item job indices are relative to the wave)
  const int2* items;         // [n_items] work items (job, strip) in dispatch order (see plan_build)
  int n_items;
  // database shard
  const int* Lt;             // [n_targets]
  // plan: the job-interleaved operand stream, [job][column 1..Lmax][k 0..6][lane] float4 (lanes shorter than
  // the job repeat their last column; the cells computed there are never used)
  const float4* jcols;
  // plan
  int njobs;
  const int* job_target;     // [njobs*32] target id (padded lanes repeat a valid id)
  uint32_t* bt;              // packed backtrace words
  struct BndSlot* bnd;       // boundary hand-off slots [job][col][32 lanes], 40 B each (see BndSlot)
  uint32_t tag_base;         // run epoch << 12; slot tag = tag_base + strip + 1
  unsigned int* counter;     // work-item queue head
  float* strip_score;        // [njobs*nstrips*32]
  int* strip_ij;             // [njobs*nstrips*32]  (i<<16 | j)
  const uint32_t* celloff;   // [sum over jobs nstrips*(Lmax+1)*32] bit r = row i0+1+r off, or null
  const float* S33;          // [44*44] or null
  // scoring
  float egq, egt, shift, ssw;
  uint32_t zero;            // always 0, opaque to the compiler (register-liveness anchor)
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// log2f4 (src/hhutil-inl.h:509-541), degree-4 minimax, unfused.  x >= 0.
// The exponent int->float conversion uses the exact magic-number form (no I2F on the hot path):
// bits(8388608.0f) + eb is the float 8388608+eb; subtracting 8388735 (=2^23+127) is exact.
__device__ __forceinline__ float log2f4_dev(float x) {
  const uint32_t u = __float_as_uint(x);
  const float e = __fadd_rn(__uint_as_float((u >> 23) | 0x4B000000u), -8388735.0f);
  const float m = __uint_as_float((u & 0x007FFFFFu) | 0x3F800000u);
  float p = -0.107254423828329604454f;
  p = __fadd_rn(__fmul_rn(p, m), 0.688243882994381274313f);
  p = __fadd_rn(__fmul_rn(p, m), -1.75647175389045657003f);
  p = __fadd_rn(__fmul_rn(p, m), 2.61761038894603480148f);
  p = __fmul_rn(p, __fadd_rn(m, -1.0f));
  return __fadd_rn(p, e);
}

// ScalarProd20Vec (src/hhviterbi.h:126-190): four partial sums r0..r3 (lane k of the reference's 4-wide
// vector sums elements k, k+4, ..., k+16), each an IEEE fp32 mul / add with round-to-nearest, i.e. exactly
// the reference's unfused sequence.
// t: the 20 target emissions as float4 x5, q: float4 x5 of the query row
__device__ __forceinline__ float dot20_dev(const float4 (&t)[5], const float4 (&q)[5]) {
  float r0 = __fmul_rn(t[0].x, q[0].x), r1 = __fmul_rn(t[0].y, q[0].y);
  float r2 = __fmul_rn(t[0].z, q[0].z), r3 = __fmul_rn(t[0].w, q[0].w);
#pragma unroll
  for (int m = 1; m < 5; ++m) {
    r0 = __fadd_rn(__fmul_rn(t[m].x, q[m].x), r0);
    r1 = __fadd_rn(__fmul_rn(t[m].y, q[m].y), r1);
    r2 = __fadd_rn(__fmul_rn(t[m].z, q[m].z), r2);
    r3 = __fadd_rn(__fmul_rn(t[m].w, q[m].w), r3);
  }
  return __fadd_rn(__fadd_rn(r0, r1), __fadd_rn(r2, r3));
}

// one 16-byte operand of the job-interleaved stream into this thread's ring slot: L2 only (a line is read once per
// strip and SM).  The data is visible to the issuing thread after its cp.async.wait_group.
__device__ __forceinline__ void cp_async_jc(float4* dst, const float4* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// operand ring of one warp: 2 column slots x 7 operands x 32 lanes (float4), i.e. one column in flight
constexpr int kJcSlot = 7 * 32;                 // float4 per column slot
constexpr size_t kRingBytes = 2 * kJcSlot * 16;   // 7168 B per warp

#define HHG_NEG (-FLT_MAX)

// x with -0 replaced by +0 (x + +0 under round-to-nearest); every other value unchanged
__device__ __forceinline__ float pos_zero(float x) { return __fadd_rn(x, 0.0f); }

// the sign bits of a (row r) and b (row r+1) as 0x00 / 0xFF bytes: selector nibble 0xB (0xF) puts the replicated msb
// of byte 3 of a (of b) in its byte.  Inline PTX because __byte_perm drops the replicate bit of a selector nibble
__device__ __forceinline__ uint32_t sign_bytes(float a, float b, uint32_t sel) {
  uint32_t p;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(p) : "r"(__float_as_uint(a)), "r"(__float_as_uint(b)), "r"(sel));
  return p;
}

// ---------------------------------------------------------------------------------------------
// Forward pass.  R rows per strip (multiple of 4).  LOCAL: par.loc.  SS: PRED_PRED ss term.
// CELLOFF: cell-off bit input (alternative alignments / excluded regions).
// ---------------------------------------------------------------------------------------------
template <int R, bool LOCAL, bool SS, bool CELLOFF>
__global__ void __launch_bounds__(kWarpsPerCta * 32, (R <= 12) ? 3 : 2)   // register caps 168 / 255 of the 64 K-register file
    k_viterbi(const VitParams P) {
  static_assert(R % 4 == 0, "R must be a multiple of 4");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // smem carve-up: [warps][R] query records | [warps] operand rings | mbarriers | (SS) the S33 table
  float4* qs = reinterpret_cast<float4*>(smem_raw) + (size_t)warp * R * 7;
  constexpr size_t kRingOff = (size_t)kWarpsPerCta * R * 112;
  // this lane's elements of the warp's ring: operand k of slot x at ring[x * kJcSlot + k * 32]
  float4* ring = reinterpret_cast<float4*>(smem_raw + kRingOff + (size_t)warp * kRingBytes) + lane;
  constexpr size_t kBarOff = kRingOff + kWarpsPerCta * kRingBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + kBarOff);
  float* s33 = reinterpret_cast<float*>(smem_raw + kBarOff + 64);
  uint64_t* bar = bars + warp;

  if (lane == 0) mbar_init(bar, 1);
  if (SS) {
    for (int k = threadIdx.x; k < 44 * 44; k += blockDim.x) s33[k] = P.S33[k];
  }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();

  const float smin = LOCAL ? 0.0f : HHG_NEG;
  const int total_items = P.n_items;
  uint32_t parity = 0;

  for (;;) {
    int item = 0;
    if (lane == 0) item = (int)atomicAdd(P.counter, 1u);
    item = __shfl_sync(0xffffffffu, item, 0);
    if (item >= total_items) break;
    // the item table is ordered group by group; inside a group of G jobs strip-major, so the strips s and s+1 of
    // one job are dispatched G items apart (natural skew) while the group's targets stay L2-resident
    const int2 it = __ldg(P.items + item);
    const int job = it.x, s = it.y;
    // job fields are read where they are used: a copy of the whole JobDesc would keep its offsets live across the
    // column loop
    const JobDesc* jd = P.jobs + job;
    const int Lq = jd->Lq;
    const int nstrips = jd->nstrips;
    const int i0 = s * R;

    // ---- stage this strip's query rows with one TMA bulk copy
    if (lane == 0) {
      mbar_expect_tx(bar, R * 112);
      tma_bulk_g2s(qs, P.qrec + (size_t)(jd->qrow0 + i0) * 7, R * 112, bar);
    }

    const int t = P.job_target[job * 32 + lane];
    const int Lt = P.Lt[t];
    const int Lmax = jd->Lmax;
    // per-column pointers advance by constants: the operand stream by 7 x 32 float4, slots and backtrace words by 32.
    // The plan allocates one column of slack after the last job's stream and slots, so the copy of column j+1 into
    // the ring needs no clamp (what it reads after the job's last column is never used)
    const float4* jc = P.jcols + jd->jc_off + lane;   // operand k of the prefetched column: jc[k*32]
    const size_t bt_row_stride = (size_t)(Lmax + 1) * 32;   // words per 4-row group
    uint32_t* btc = P.bt + jd->bt_off + lane + (size_t)(i0 >> 2) * bt_row_stride + 32;   // column j
    BndSlot* bndc = P.bnd + jd->bnd_off + 32;          // the job's 32 slots of column j
    const uint32_t tag_in = P.tag_base + (uint32_t)s;        // written by strip s-1
    const uint32_t tag_out = P.tag_base + (uint32_t)s + 1u;  // what this strip writes
    const bool last_strip = (s == nstrips - 1);
    const uint32_t* co = nullptr;                            // column j
    if (CELLOFF) co = P.celloff + jd->co_off + (size_t)s * (Lmax + 1) * 32 + lane + 32;

    // ---- state of the R rows at the previous column (column 0 initially), :161-173.
    // Every array element is read by its own row before the row overwrites it, so the state updates in place:
    //   * MI is not kept.  Its two readers are row r+1's c5 at column j+1 (diagonal) and row r+1's mi at column j
    //     (up), and both add q_m2m(r+1) first; Y[r] = MI(r-1, j-1) + q_m2m(r) is that shared sum.
    //   * the other diagonal reads (c1..c4 of row r+1) take partial sums that row r forms from its old values
    //     before it overwrites them (pMM, pGD, pIM, pDG).
    // The gap-state flags read sign bits and need every DP value to differ from -0 (see the row body).  -i·egq and
    // -j·egt are -0 when a gap cost is 0, so the boundary values take +0 for -0 (pos_zero).
    float MM[R], GD[R], IM[R], DG[R], Y[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
      MM[r] = pos_zero(__fmul_rn((float)(-(i0 + 1 + r)), P.egq));
      GD[r] = IM[r] = DG[r] = HHG_NEG;
    }
    // boundary row i0 at column j-1 (diagonal of the strip's first row)
    float dtMM = pos_zero(__fmul_rn((float)(-i0), P.egq)), dtDG = HHG_NEG, dtGD = HHG_NEG, dtIM = HHG_NEG;

    float best = HHG_NEG;
    int bi = 0, bj = 0;

    // first column into ring slot 0 (Lmax >= 1); column j lives in slot (j - 1) & 1
#pragma unroll
    for (int k = 0; k < 7; ++k) cp_async_jc(ring + k * 32, jc + k * 32);
    cp_async_commit();
    int rd = 0;   // float4 offset of column j's slot

    // boundary values of column 1 (strips > 0): issue the slot load now, validate the tag at use
    float nMM = 0.f, nDG = 0.f, nMI = 0.f, nGD = 0.f, nIM = 0.f;
    uint32_t ntag[5] = {0u, 0u, 0u, 0u, 0u};
    if (s > 0) ld_slot(bndc, lane, nMM, nDG, nMI, nGD, nIM, ntag);

    mbar_wait(bar, parity);
    parity ^= 1u;
#pragma unroll
    for (int r = 0; r < R; ++r) Y[r] = __fadd_rn(HHG_NEG, qs[r * 7 + 5].x);   // MI(., 0) = -FLT_MAX

    for (int j = 1; j <= Lmax; ++j) {
      // ---- current column operands from the ring, then the copy of the next column into the other slot.  That slot
      // held column j-1, whose LDS results column j-1 has already consumed, so the copy cannot overwrite unread data
      cp_async_wait_all();
      const float4* cur = ring + rd;
      const float4 tp[5] = {cur[0], cur[32], cur[64], cur[96], cur[128]};
      const float4 tt0 = cur[160], tt1 = cur[192];
      const float t_m2m = tt0.x, t_m2d = tt0.y, t_d2m = tt0.z, t_d2d = tt0.w;
      const float t_i2m = tt1.x, t_i2i = tt1.y, t_m2i = tt1.z;
      const uint32_t t_ss = __float_as_uint(tt1.w);
      rd ^= kJcSlot;
      jc += 224;
#pragma unroll
      for (int k = 0; k < 7; ++k) cp_async_jc(ring + rd + k * 32, jc + k * 32);
      cp_async_commit();

      // ---- boundary row i0 at column j: slot prefetched during column j-1; wait until the producer strip's
      // tag is there, then prefetch column j+1
      float tMM, tDG, tMI, tGD, tIM;
      if (s == 0) {
        tMM = pos_zero(__fmul_rn((float)(-j), P.egt));   // :148
        tDG = tMI = tGD = tIM = HHG_NEG;
      } else {
        // all five words must carry the producer's tag.  One warp vote on the common path; strip s-1 normally runs
        // ahead, so the per-lane retry loop is rare
        if (!__all_sync(0xffffffffu, slot_ok(ntag, tag_in))) {
          while (!slot_ok(ntag, tag_in)) {
            __nanosleep(20);
            ld_slot(bndc, lane, nMM, nDG, nMI, nGD, nIM, ntag);
          }
        }
        tMM = nMM; tDG = nDG; tMI = nMI; tGD = nGD; tIM = nIM;
        ld_slot(bndc + 32, lane, nMM, nDG, nMI, nGD, nIM, ntag);
      }
      uint32_t cow = 0;
      if (CELLOFF) cow = __ldg(co);

      // row 0's diagonal partial sums from the boundary row at column j-1; row r+1's are formed by row r
      float4 qa = qs[5], qb = qs[6];
      float pMM = __fadd_rn(dtMM, qa.x), pGD = __fadd_rn(dtGD, qa.x), pIM = __fadd_rn(dtIM, qb.x),
            pDG = __fadd_rn(dtDG, qa.z);
      float uMM = tMM, uDG = tDG, uMI = tMI;                              // cell (i-1, j)
      const float bcmp = (j <= Lt) ? best : INFINITY;   // padded columns never become the maximum
      float bc = bcmp;

      // The trace word of 4 rows starts at 6 in every byte and takes each row's MM code XOR 6 by XOR (see b below).
      // (t_ss & P.zero) is 0; it only keeps the 4th register of the operand LDS.128 live (see ld_slot)
      constexpr uint32_t kWord0 = 0x06060606u;
      uint32_t word = kWord0 ^ (SS ? 0u : (t_ss & P.zero));
      uint32_t eb = 0u;                                     // b of the pair's even row
      float eGD = 0.f, eIM = 0.f, eDG = 0.f, eMI = 0.f;   // and its gap-flag differences
#pragma unroll
      for (int r = 0; r < R; ++r) {
        float4 q[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) q[k] = qs[r * 7 + k];
        const float q_m2m = qa.x, q_m2d = qa.y, q_d2m = qa.z, q_d2d = qa.w;
        const float q_i2m = qb.x, q_i2i = qb.y, q_m2i = qb.z;
        const uint32_t q_ss = __float_as_uint(qb.w);
        const int sh = 8 * (r & 3);   // this row's byte of the trace word

        // 5-way maximum with the reference's strict-'>' / first-wins rule, :241-273.  b is the MM code XOR 6, already
        // in this row's byte: code 6 (MI) becomes 0, so every select of the chain has one constant and no MOV
        uint32_t b;
        float mm;
        const float c1 = __fadd_rn(pMM, t_m2m);     // (MM(i-1,j-1) + q_m2m) + t_m2m
        const float c2 = __fadd_rn(pGD, t_d2m);     // (GD(i-1,j-1) + q_m2m) + t_d2m
        const float c3 = __fadd_rn(pIM, t_m2m);     // (IM(i-1,j-1) + q_i2m) + t_m2m
        const float c4 = __fadd_rn(pDG, t_m2m);     // (DG(i-1,j-1) + q_d2m) + t_m2m
        const float c5 = __fadd_rn(Y[r], t_i2m);    // (MI(i-1,j-1) + q_m2m) + t_i2m
#if HHG_MAX3
        // the winner of the strict-'>' chain is the FIRST candidate (order STOP, MM, GD, IM, DG, MI) that attains
        // the maximum: five maxima + five equality selects instead of five max + five '>' selects
        mm = fmaxf(fmaxf(smin, c1), c2);
        mm = fmaxf(fmaxf(mm, c3), c4);
        mm = fmaxf(mm, c5);
        b = (c4 == mm) ? (5u ^ 6u) << sh : 0u;
        b = (c3 == mm) ? (4u ^ 6u) << sh : b;
        b = (c2 == mm) ? (3u ^ 6u) << sh : b;
        b = (c1 == mm) ? (2u ^ 6u) << sh : b;
        b = (smin == mm) ? (0u ^ 6u) << sh : b;
#else
        b = (c1 > smin) ? (2u ^ 6u) << sh : 6u << sh; mm = fmaxf(smin, c1);
        b = (c2 > mm) ? (3u ^ 6u) << sh : b;          mm = fmaxf(mm, c2);
        b = (c3 > mm) ? (4u ^ 6u) << sh : b;          mm = fmaxf(mm, c3);
        b = (c4 > mm) ? (5u ^ 6u) << sh : b;          mm = fmaxf(mm, c4);
        b = (c5 > mm) ? 0u : b;                       mm = fmaxf(mm, c5);
#endif

        float Si = log2f4_dev(dot20_dev(tp, q));                     // :277
        if (SS) {
          Si = __fadd_rn(__fmul_rn(P.ssw, s33[q_ss * 44 + t_ss]), Si);   // :210,279
        }
        Si = __fadd_rn(Si, P.shift);                                   // :281
        mm = __fadd_rn(mm, Si);

        const float oMM = MM[r], oGD = GD[r], oIM = IM[r], oDG = DG[r];   // (i, j-1)
        // the next row's diagonal partial sums, from this row's old values and before its new ones: with no old value
        // live past its replacement ptxas keeps each state in one register (otherwise ~40 copies per column)
        if (r + 1 < R) {
          qa = qs[(r + 1) * 7 + 5]; qb = qs[(r + 1) * 7 + 6];
          pMM = __fadd_rn(oMM, qa.x); pGD = __fadd_rn(oGD, qa.x); pIM = __fadd_rn(oIM, qb.x);
          pDG = __fadd_rn(oDG, qa.z);
        }
        // Gap-state flags.  The reference's a1 > a2 is the sign bit of a2 - a1 (an FADD instead of a compare and a
        // select on the integer pipe): a difference of two floats is 0 only when they are equal, overflow and
        // underflow keep the sign, and the canonical NaN of -inf - -inf or inf - inf has a clear sign bit, as a1 > a2
        // is false there.  The one exception, (-0) - (+0) = -0, cannot occur: under round-to-nearest a sum is -0 only
        // when both addends are -0, every sum here and in the MM recurrence has an addend that is a DP value, Si or
        // -FLT_MAX, and so by induction no DP value is -0 once the boundary values are not (pos_zero above).  Si is
        // never -0: log2f4's e is an exact difference, +0 when it vanishes.  Transitions may be -0.
        float a1, a2, gd, im, dg, mi, dGD, dIM, dDG, dMI;
        a1 = __fadd_rn(oMM, t_m2d); a2 = __fadd_rn(oGD, t_d2d);                                // :307
        dGD = __fsub_rn(a2, a1); gd = fmaxf(a1, a2);
        a1 = __fadd_rn(__fadd_rn(oMM, q_m2i), t_m2m); a2 = __fadd_rn(__fadd_rn(oIM, q_i2i), t_m2m);   // :324
        dIM = __fsub_rn(a2, a1); im = fmaxf(a1, a2);
        a1 = __fadd_rn(uMM, q_m2d); a2 = __fadd_rn(uDG, q_d2d);                                // :340
        dDG = __fsub_rn(a2, a1); dg = fmaxf(a1, a2);
        Y[r] = __fadd_rn(uMI, q_m2m);                                                           // c5 of column j+1
        a1 = __fadd_rn(__fadd_rn(uMM, q_m2m), t_m2i); a2 = __fadd_rn(Y[r], t_i2i);             // :358
        dMI = __fsub_rn(a2, a1); mi = fmaxf(a1, a2);

        if (CELLOFF) {                                                 // :373-392
          const float off = ((cow >> r) & 1u) ? HHG_NEG : 0.0f;
          mm = __fadd_rn(mm, off); gd = __fadd_rn(gd, off); im = __fadd_rn(im, off);
          dg = __fadd_rn(dg, off); mi = __fadd_rn(mi, off);
        }

        // rows r-1 and r go into their bytes together: one LOP3 for both MM codes, and per flag one PRMT and one LOP3
        if (r & 1) {
          const int q = r & 2;   // byte of row r-1
          const uint32_t sel = 0xFBu << (4 * q);
          word ^= eb ^ b;
          word |= sign_bytes(eGD, dGD, sel) & (0x0808u << (8 * q));
          word |= sign_bytes(eIM, dIM, sel) & (0x1010u << (8 * q));
          word |= sign_bytes(eDG, dDG, sel) & (0x2020u << (8 * q));
          word |= sign_bytes(eMI, dMI, sel) & (0x4040u << (8 * q));
        } else {
          eb = b; eGD = dGD; eIM = dIM; eDG = dDG; eMI = dMI;
        }
        if ((r & 3) == 3) {
          __stcs(btc + (size_t)(r >> 2) * bt_row_stride, word);
          word = kWord0;
        }
        // this row's new values are the next row's up
        uMM = mm; uDG = dg; uMI = mi;
        MM[r] = mm; GD[r] = gd; IM[r] = im; DG[r] = dg;
      }
      dtMM = tMM; dtDG = tDG; dtGD = tGD; dtIM = tIM;

      // running maximum, :423-455: ONE test per column on the maximum m of the R new MM values (a tree of
      // FMNMX, 1 instruction per row instead of compare+branch per cell).  Strips are swept column-major, the
      // reference row-major: on an exact tie the earlier ROW must win (mm == best && i < bi).
      {
        float c0 = MM[0], c1 = MM[1], c2 = MM[2], c3 = MM[3];   // four interleaved chains (R is a multiple of 4)
#pragma unroll
        for (int r = 4; r < R; r += 4) {
          c0 = fmaxf(c0, MM[r]); c1 = fmaxf(c1, MM[r + 1]); c2 = fmaxf(c2, MM[r + 2]); c3 = fmaxf(c3, MM[r + 3]);
        }
        const float m = fmaxf(fmaxf(c0, c1), fmaxf(c2, c3));
        if (LOCAL) {
          // every row up to Lq is a candidate: the column's record is its argmax, the FIRST row that reaches the
          // maximum, taken when it beats the strip's best or ties it at a smaller row.  A warp vote skips the select
          // chain on columns where no lane can move; the chain and the update are predicated, with no per-row branch.
          // The maximum's bits are the row's: MM is never -0 (its last FADD adds Si, which is never -0).
          if (__any_sync(0xffffffffu, m >= bcmp)) {
            float mc = m;
            if (i0 + R > Lq) {   // the last strip of a query that is not a multiple of R: rows past Lq do not count
              mc = -INFINITY;
#pragma unroll
              for (int r = 0; r < R; ++r) mc = fmaxf(mc, (i0 + 1 + r <= Lq) ? MM[r] : -INFINITY);
            }
            int r1 = R - 1;
#pragma unroll
            for (int r = R - 2; r >= 0; --r) r1 = (MM[r] == mc) ? r : r1;
            const int i = i0 + 1 + r1;
            if (mc >= bcmp && (mc > best || i < bi)) { best = mc; bi = i; bj = j; }
          }
        } else if (m >= bc) {
          // global mode, where only row Lq and column Lt count: rows in ascending order
#pragma unroll
          for (int r = 0; r < R; ++r) {
            const float mm = MM[r];
            if (mm >= bc) {
              const int i = i0 + 1 + r;
              const bool cand = (i <= Lq) && (LOCAL || i == Lq || j == Lt);
              if (cand && (mm > best || i < bi)) { best = mm; bi = i; bj = j; bc = mm; }
            }
          }
        }
      }

      if (!last_strip) st_slot(bndc, lane, uMM, uDG, uMI, GD[R - 1], IM[R - 1], tag_out);
      bndc += 32;
      btc += 32;
      if (CELLOFF) co += 32;
    }
    // the job's address is formed again from the opaque index: reusing jd would keep that 64-bit pointer live across
    // the column loop, and that loop measured 0.8 % slower at R = 16 (H100 80GB HBM3, 700 W power limit)
    int jb = job;
    asm("" : "+r"(jb));
    const size_t o = ((size_t)P.jobs[jb].ss_off + s) * 32 + lane;
    P.strip_score[o] = best;
    P.strip_ij[o] = (bi << 16) | bj;
    // the copy of column Lmax+1 (slack, never read) must land before the next item's first copy targets the ring
    cp_async_wait_all();
    __syncwarp();   // all lanes done with the smem slice before the next TMA overwrites it
  }
}

// pnul[a] of HMM::IncludeNullModelInHMM (src/hhhmm.cpp:2059-2088) for one (query, template) pair.
// columnscore: 0 = pb, 1 = 0.5(q.pav + t.pav) (default), 2 = t.pav, 3 = q.pav.
__device__ __forceinline__ void null_model_vec(int columnscore, const float* __restrict__ q_pav,
                                               const float* __restrict__ t_pav, const float* __restrict__ pb,
                                               float (&pn)[20]) {
#pragma unroll
  for (int a = 0; a < 20; ++a) {
    switch (columnscore) {
      case 0: pn[a] = pb[a]; break;
      case 2: pn[a] = t_pav[a]; break;
      case 3: pn[a] = q_pav[a]; break;
      default: pn[a] = __fmul_rn(0.5f, __fadd_rn(q_pav[a], t_pav[a])); break;
    }
  }
}
__device__ __forceinline__ float4 div4(float4 v, const float* pn) {
  v.x = __fdiv_rn(v.x, pn[0]); v.y = __fdiv_rn(v.y, pn[1]); v.z = __fdiv_rn(v.z, pn[2]); v.w = __fdiv_rn(v.w, pn[3]);
  return v;
}

// ---------------------------------------------------------------------------------------------
// Backtrace: one thread per requested target.  Merges the per-strip maxima in row order (strict '>',
// i.e. the reference's row-major first-occurrence rule) and walks the packed byte matrix.
// ---------------------------------------------------------------------------------------------
struct HitRec {
  float score;
  int i2, j2, i1, j1, nsteps, matched_cols, path_off;
  float hit_score;   // Hit.score: Viterbi score - ss score + correlation term (src/hhviterbi.cpp:215-256)
  float score_ss;    // Hit.score_ss
};

struct BtParams {
  int n_req;
  const JobDesc* jobs;       // [njobs] all of the plan's jobs (absolute job index)
  const ReqDesc* reqs;       // [n_req]
  // fused null model (query-batch plans over a raw shard): cols = emissions BEFORE the null model and the division
  // t.p[j][a] / pnul[a] is applied on the fly exactly like HMM::IncludeNullModelInHMM; nm_mode < 0: cols are prepared
  int nm_mode;
  const float* q_pav;        // [nq*20]
  const float* t_pav;        // [n_targets*20]
  const float* pb;           // [20]
  int job_begin, job_end;    // only requests whose job lies in [job_begin, job_end) are traced
  const uint32_t* bt;
  const float* strip_score;
  const int* strip_ij;
  HitRec* hits;
  uint8_t* paths;            // may be null
  // Hit.score (Viterbi::ScoreForBacktrace, src/hhviterbi.cpp:195-281)
  const float4* qrec;        // query row records (p in the first 5 float4)
  const float4* cols;        // target column records
  const long long* col_off;
  const float* lg2;          // fast_log2 tables (src/util-inl.h:108-128): lg2[1025], diff[1025]
  const float* diff;
  const float* S33;          // may be null
  float* S;                  // [path_total] per-step column scores (scratch)
  float corr, ssw;
  int use_ss;                // PRED_PRED ss term was part of the alignment score
  int ss_score_mode;         // par.ssm == 2: subtract the ss score again (SCORE_ALIGNMENT)
};

// Score(q.p[i], t.p[j]) = fast_log2(ScalarProd20(q, t)), src/hhhit-inl.h:61-134.  In the AVX2 build of the
// reference (the pinned oracle) the macro SSE is not defined in that header, so ScalarProd20 is the
// plain left-to-right sum  t0*q0 + t1*q1 + ... + t19*q19  (verified against the compiled reference:
// 300/300 random vectors bit-identical; the SSE shuffle tree matches only ~70%).
__device__ __forceinline__ float score_cols_dev(const float4* q, const float4* t, const float* lg2,
                                                const float* diff, const float* pn = nullptr) {
  float sum = 0.0f;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    const float4 a = q[k];
    const float4 b = pn ? div4(t[k], pn + 4 * k) : t[k];
    if (k == 0) sum = __fmul_rn(b.x, a.x); else sum = __fadd_rn(sum, __fmul_rn(b.x, a.x));
    sum = __fadd_rn(sum, __fmul_rn(b.y, a.y));
    sum = __fadd_rn(sum, __fmul_rn(b.z, a.z));
    sum = __fadd_rn(sum, __fmul_rn(b.w, a.w));
  }
  return fast_log2_dev(sum, lg2, diff);
}

__device__ __forceinline__ uint32_t bt_byte(const uint32_t* btj, size_t row_stride, int i, int j) {
  const uint32_t w = btj[(size_t)((i - 1) >> 2) * row_stride + (size_t)j * 32];
  return (w >> (8 * ((i - 1) & 3))) & 0xFFu;
}

__global__ void k_backtrace(const BtParams P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.n_req) return;
  const ReqDesc rq = P.reqs[k];
  const int job = rq.job, lane = rq.lane;
  if (job < P.job_begin || job >= P.job_end) return;
  const JobDesc jd = P.jobs[job];
  float best = HHG_NEG;
  int ij = 0;
  for (int s = 0; s < jd.nstrips; ++s) {
    const size_t o = ((size_t)jd.ss_off + s) * 32 + lane;
    const float v = P.strip_score[o];
    if (v > best) { best = v; ij = P.strip_ij[o]; }
  }
  const int i2 = ij >> 16, j2 = ij & 0xFFFF;
  const uint32_t* btj = P.bt + jd.bt_off + lane;
  const size_t rs = (size_t)(jd.Lmax + 1) * 32;
  uint8_t* path = P.paths ? P.paths + rq.path_off : nullptr;

  const float4* tcol = P.cols + (size_t)P.col_off[rq.target] * 7;
  const float4* qrec = P.qrec + (size_t)jd.qrow0 * 7;
  float pnv[20];
  const float* pn = nullptr;
  if (P.nm_mode >= 0) {
    null_model_vec(P.nm_mode, P.q_pav + (size_t)jd.query * 20, P.t_pav + (size_t)rq.target * 20, P.pb, pnv);
    pn = pnv;
  }
  float* S = P.S + rq.path_off;
  float score_ss = 0.0f;

  int step = 0, i = i2, j = j2, mc = 0, li = i2, lj = j2;
  int state = 2;   // MM
  while (state != 0) {
    if (path) path[step] = (uint8_t)state;
    // per-step column score: only MM steps score (src/hhviterbi.cpp:219-235); the step that turns out to
    // be the last one is re-scored below because the reference forces states[nsteps] = MM first
    float Sv = 0.0f;
    if (state == 2 && i >= 1 && j >= 1) {
      Sv = score_cols_dev(qrec + (size_t)(i - 1) * 7, tcol + (size_t)(j - 1) * 7, P.lg2, P.diff, pn);
      if (P.use_ss) {
        const uint32_t qs = __float_as_uint(qrec[(size_t)(i - 1) * 7 + 6].w);
        const uint32_t ts = __float_as_uint(tcol[(size_t)(j - 1) * 7 + 6].w);
        score_ss = __fadd_rn(score_ss, __fmul_rn(P.ssw, P.S33[qs * 44 + ts]));
      }
    }
    S[step] = Sv;
    ++step;
    li = i; lj = j;
    const uint32_t c = (i >= 1 && j >= 1) ? bt_byte(btj, rs, i, j) : 0u;
    const int prev_state = state;
    switch (state) {
      case 2: ++mc; state = (i <= 1 || j <= 1) ? 0 : (int)(c & 7u); --i; --j; break;
      case 3: if (j <= 1) state = 0; else { if (c & 8u) state = 2; --j; } break;
      case 4: if (j <= 1) state = 0; else { if (c & 16u) state = 2; --j; } break;
      case 5: if (i <= 1) state = 0; else { if (c & 32u) state = 2; --i; } break;
      case 6: if (i <= 1) state = 0; else { if (c & 64u) state = 2; --i; } break;
      default: state = 0; break;
    }
    if (state == 0 && prev_state != 2 && li >= 1 && lj >= 1) {
      // last step ended in a gap state: the reference relabels it MM (src/hhviterbi.cpp:147) and scores it
      S[step - 1] = score_cols_dev(qrec + (size_t)(li - 1) * 7, tcol + (size_t)(lj - 1) * 7, P.lg2, P.diff, pn);
      if (P.use_ss) {
        const uint32_t qs = __float_as_uint(qrec[(size_t)(li - 1) * 7 + 6].w);
        const uint32_t ts = __float_as_uint(tcol[(size_t)(lj - 1) * 7 + 6].w);
        score_ss = __fadd_rn(score_ss, __fmul_rn(P.ssw, P.S33[qs * 44 + ts]));
      }
    }
  }
  if (path && step > 0) path[step - 1] = 2;   // states[nsteps] = MM, src/hhviterbi.cpp:147
  // Hit.score, src/hhviterbi.cpp:237-256: four correlation passes in the reference's order
  float hs = best;
  if (P.ss_score_mode) hs = __fadd_rn(hs, -score_ss);
  float scorr = 0.0f;
  if (step > 0) {
    for (int d = 1; d <= 4; ++d)
      for (int st = d; st < step; ++st) scorr = __fadd_rn(scorr, __fmul_rn(S[st], S[st - d]));
    hs = __fadd_rn(hs, __fmul_rn(P.corr, scorr));
  }
  HitRec h;
  h.score = best; h.i2 = i2; h.j2 = j2; h.i1 = li; h.j1 = lj; h.nsteps = step;
  h.matched_cols = mc; h.path_off = (int)rq.path_off;
  h.hit_score = hs; h.score_ss = score_ss;
  P.hits[k] = h;
}

// Query-dependent part of PrepareTemplateHMM: factor the null model into the template emissions
// (HMM::IncludeNullModelInHMM, src/hhhmm.cpp:2059-2088).  One thread per target column; exact fp32
// division like the reference.  columnscore: 0 = pb, 1 = 0.5(q.pav + t.pav) (default), 2 = t.pav, 3 = q.pav.
__global__ void k_null_model(long long total_cols, int n, const long long* col_off, const float4* raw,
                             const float* t_pav, const float* q_pav, const float* pb, int columnscore,
                             float4* out) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= total_cols) return;
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (col_off[mid] <= c) lo = mid; else hi = mid - 1;
  }
  float pn[20];
  null_model_vec(columnscore, q_pav, t_pav + (size_t)lo * 20, pb, pn);
  const float4* src = raw + (size_t)c * 7;
  float4* dst = out + (size_t)c * 7;
#pragma unroll
  for (int k = 0; k < 5; ++k) dst[k] = div4(src[k], pn + 4 * k);
  dst[5] = src[5];
  dst[6] = src[6];
}

// Template records of a MAC realignment over a raw shard (hhg_mac_realign_batch): request r's Lt[r] records are
// copied from the raw records of target[r] into out + dst[r] (both in records), with the null model of its query
// req_q[r] factored into the emissions by the same operations as k_null_model.  The realignment then reads its own
// copy, whatever query hhg_db_apply_null_model last prepared the shard's `cols` for.  Grid: (x, requests).
__global__ void k_mac_gather_cols(int n, const int* __restrict__ req_q, const int* __restrict__ target,
                                  const int* __restrict__ Lt, const long long* __restrict__ col_off,
                                  const long long* __restrict__ dst, const float4* __restrict__ raw,
                                  const float* __restrict__ t_pav, const float* __restrict__ q_pav,
                                  const float* __restrict__ pb, int columnscore, float4* __restrict__ out) {
  const int r = blockIdx.y;
  if (r >= n) return;
  const int t = target[r], L = Lt[r];
  float pn[20];
  null_model_vec(columnscore, q_pav + (size_t)req_q[r] * 20, t_pav + (size_t)t * 20, pb, pn);
  const float4* src0 = raw + (size_t)col_off[t] * 7;
  float4* dst0 = out + (size_t)dst[r] * 7;
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < L; c += gridDim.x * blockDim.x) {
    const float4* src = src0 + (size_t)c * 7;
    float4* d = dst0 + (size_t)c * 7;
#pragma unroll
    for (int k = 0; k < 5; ++k) d[k] = div4(src[k], pn + 4 * k);
    d[5] = src[5];
    d[6] = src[6];
  }
}

// Staging of a host-resident store's targets into a staged shard (hhg_db_stage): descriptor d copies the len records
// at store record src to arena record dst and fills slot's entries of L, col_off and pav; len == 0 marks a slot that
// lost its target (only L is cleared).  `store` and `store_pav` are device-mapped page-locked HOST memory, so every
// load crosses the PCIe link: latency, not SM throughput, bounds the copy.  A work item is one run of kStageRun records
// of one target (a target's records are contiguous on both sides, a long target is several items, the last one short);
// a warp takes an item, finds its target by bisection over run0 (first item of each descriptor) and every lane issues
// its kStageRun * 7 / 32 independent 16-byte loads -- read once, so they bypass L1 -- before its first store.  A few
// dozen warps keep more bytes in flight than the link's bandwidth-delay product, so the grid is small and the kernel
// can share the device with a search running on another stream.
constexpr int kStageRun = 32;                      // records per work item: 3584 B, 7 x 16 B per lane
struct __align__(16) StageDesc {
  long long src, dst;
  int len, slot, global, run0;
};
static_assert(sizeof(StageDesc) == 32, "StageDesc is two 16-byte words");

__device__ __forceinline__ float4 ld_stream(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

__global__ void __launch_bounds__(256)
k_stage_gather(int n_desc, int n_runs, const StageDesc* __restrict__ desc, const float4* __restrict__ store,
               const float* __restrict__ store_pav, float4* __restrict__ cols_raw, float* __restrict__ pav,
               int* __restrict__ L, long long* __restrict__ col_off) {
  constexpr int kPer = kStageRun * 7 / 32;
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (int run = warp; run < n_runs; run += nwarps) {
    int lo = 0, hi = n_desc - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (desc[mid].run0 <= run) lo = mid; else hi = mid - 1;
    }
    const StageDesc d = desc[lo];
    const int r0 = (run - d.run0) * kStageRun;
    const int nvec = min(kStageRun, d.len - r0) * 7;
    const float4* src = store + (size_t)(d.src + r0) * 7;
    float4* dst = cols_raw + (size_t)(d.dst + r0) * 7;
    float4 v[kPer];
#pragma unroll
    for (int k = 0; k < kPer; ++k)
      if (lane + 32 * k < nvec) v[k] = ld_stream(src + lane + 32 * k);
#pragma unroll
    for (int k = 0; k < kPer; ++k)
      if (lane + 32 * k < nvec) dst[lane + 32 * k] = v[k];
  }
  // per-target entries: 5 lanes per descriptor move the 20 floats of pav, the first also writes L and col_off
  for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < n_desc * 8; w += gridDim.x * blockDim.x) {
    const StageDesc d = desc[w >> 3];
    const int part = w & 7;
    if (part == 0) {
      L[d.slot] = d.len;
      if (d.len) col_off[d.slot] = d.dst;
    }
    if (d.len && part < 5)
      reinterpret_cast<float4*>(pav + (size_t)d.slot * 20)[part] =
          ld_stream(reinterpret_cast<const float4*>(store_pav + (size_t)d.global * 20) + part);
  }
}

// Compact the per-request path strings (capacity Lq+Lt+2 each) to their real lengths before the D2H copy:
// one thread per request copies nsteps bytes to its compact offset.
__global__ void k_gather_paths(int n, const HitRec* hits, const ReqDesc* reqs, const long long* dst_off,
                               const uint8_t* src, uint8_t* dst) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int len = hits[k].nsteps;
  const uint8_t* s = src + reqs[k].path_off;
  uint8_t* d = dst + dst_off[k];
  for (int b = 0; b < len; ++b) d[b] = s[b];
}

// De-interleave one target's backtrace bytes into the reference's row-major cell matrix (parity tests).
__global__ void k_debug_bt(const uint32_t* bt, long long bt_off, int lane, int Lmax, int Lq, int Lt,
                           uint8_t* out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = (Lq + 1) * (Lt + 1);
  if (idx >= total) return;
  const int i = idx / (Lt + 1), j = idx - i * (Lt + 1);
  uint8_t v = 0;
  if (i >= 1 && j >= 1) v = (uint8_t)bt_byte(bt + bt_off + lane, (size_t)(Lmax + 1) * 32, i, j);
  out[idx] = v;
}

// Pack prepared profiles (include/hhg.h layout) into column records: thread per (target, column).
__global__ void k_pack_cols(int n, const int* L, const long long* col_off, const long long* p_off,
                            const long long* tr_off, const long long* ss_off, const float* p,
                            const float* tr, const uint8_t* ss, ColRec* out, long long total_cols) {
  const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= total_cols) return;
  // binary search the target owning column c
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (col_off[mid] <= c) lo = mid; else hi = mid - 1;
  }
  const int t = lo;
  const int j = (int)(c - col_off[t]) + 1;   // 1-based column
  const float* pp = p + p_off[t] + (size_t)j * 20;
  const float* t1 = tr + tr_off[t] + (size_t)(j - 1) * 7;
  const float* t0 = tr + tr_off[t] + (size_t)j * 7;
  ColRec r;
#pragma unroll
  for (int a = 0; a < 20; ++a) r.p[a] = pp[a];
  r.m2m = t1[0]; r.m2d = t1[2]; r.d2m = t1[5]; r.d2d = t1[6]; r.i2m = t1[3];
  r.i2i = t0[4]; r.m2i = t0[1];
  r.ss = ss ? (uint32_t)ss[ss_off[t] + j] : 0u;
  out[c] = r;
}

// Build the job-interleaved operand stream of a plan from the shard's column records: warp per (job, column),
// lane = the job's lane.  Each lane copies its own 112-byte record (7 x 16 B) of column min(j, Lt) into
// out[jobs[job].jc_off + ((j-1)*7 + k)*32 + lane]: the seven stores of a warp are full 512-byte lines.
__global__ void __launch_bounds__(256)
k_interleave_cols(const JobDesc* __restrict__ jobs, const int* __restrict__ job_target, const float4* __restrict__ cols,
                  const long long* __restrict__ col_off, const int* __restrict__ Lt, float4* __restrict__ out,
                  int nm_mode, const float* __restrict__ q_pav, const float* __restrict__ t_pav,
                  const float* __restrict__ pb) {
  const int job = blockIdx.x;
  const int lane = threadIdx.x & 31;
  const int Lmax = jobs[job].Lmax;
  const int t = job_target[job * 32 + lane];
  const int L = Lt[t];
  const float4* src0 = cols + (size_t)col_off[t] * 7;
  float4* dst0 = out + jobs[job].jc_off + lane;
  // nm_mode >= 0: `cols` holds the emissions before the null model; factor it in for this job's query on the way
  // (HMM::IncludeNullModelInHMM, the query-dependent step of PrepareTemplateHMM), so a batch of queries can share one
  // resident raw shard
  float pn[20];
  if (nm_mode >= 0) null_model_vec(nm_mode, q_pav + (size_t)jobs[job].query * 20, t_pav + (size_t)t * 20, pb, pn);
  for (int j = blockIdx.y * 8 + (threadIdx.x >> 5) + 1; j <= Lmax; j += gridDim.y * 8) {
    const float4* src = src0 + (size_t)(min(j, L) - 1) * 7;
    float4* dst = dst0 + (size_t)(j - 1) * 224;
#pragma unroll
    for (int k = 0; k < 5; ++k) dst[k * 32] = nm_mode >= 0 ? div4(__ldg(src + k), pn + 4 * k) : __ldg(src + k);
    dst[5 * 32] = __ldg(src + 5);
    dst[6 * 32] = __ldg(src + 6);
  }
}

// Rasterise excluded alignments into the cell-off bit words (Viterbi::ExcludeAlignment,
// src/hhviterbi.cpp:61-77): one thread per excluded path step.
__global__ void k_celloff_raster(int n_steps, const int* step_req, const int* step_i, const int* step_j,
                                 const ReqDesc* reqs, const JobDesc* jobs, int R, uint32_t* co) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_steps) return;
  const ReqDesc& rq = reqs[step_req[k]];
  const int Lt = rq.Lt, Lq = rq.Lq;
  const int Lmax = jobs[rq.job].Lmax;
  uint32_t* base = co + jobs[rq.job].co_off + rq.lane;
  const int i = step_i[k], j = step_j[k];
  const int W = 40;   // VITERBI_PATH_WIDTH, src/hhdecl.h:50
  for (int ii = max(i - W, 1); ii <= min(i + W, Lq); ++ii) {
    const int s = (ii - 1) / R, r = (ii - 1) - s * R;
    atomicOr(base + ((size_t)s * (Lmax + 1) + j) * 32, 1u << r);
  }
  for (int jj = max(j - W, 1); jj <= min(j + W, Lt); ++jj) {
    const int s = (i - 1) / R, r = (i - 1) - s * R;
    atomicOr(base + ((size_t)s * (Lmax + 1) + jj) * 32, 1u << r);
  }
}

// Excluded regions (ViterbiRunner::exclude_regions / exclude_template_regions, src/hhviterbirunner.cpp:291-330; the
// -excl / -template_excl options): query rows i0..i1 are switched off for every template column, template columns
// j0..j1 for every query row.  One thread per cell-off word (job, strip, column, lane).
__global__ void __launch_bounds__(256)
k_celloff_regions(long long n_words, int njobs, const JobDesc* __restrict__ jobs, int R, int nqr,
                  const int* __restrict__ q_lo, const int* __restrict__ q_hi, int ntr, const int* __restrict__ t_lo,
                  const int* __restrict__ t_hi, uint32_t* __restrict__ co) {
  const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_words) return;
  int lo = 0, hi = njobs - 1;                       // job owning word w
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].co_off <= w) lo = mid; else hi = mid - 1;
  }
  const long long rel = w - jobs[lo].co_off;
  const int cols1 = jobs[lo].Lmax + 1;
  const int s = (int)(rel / ((long long)cols1 * 32));
  const int j = (int)((rel / 32) % cols1);
  if (s >= jobs[lo].nstrips || j < 1) return;
  uint32_t m = 0;
  for (int k = 0; k < ntr; ++k) if (j >= t_lo[k] && j <= t_hi[k]) m = 0xFFFFFFFFu;
  for (int k = 0; k < nqr && m != 0xFFFFFFFFu; ++k) {
    const int a = max(q_lo[k], s * R + 1), b = min(q_hi[k], s * R + R);   // rows of this strip inside the range
    if (a <= b) m |= (b - a + 1 >= 32 ? 0xFFFFFFFFu : ((1u << (b - a + 1)) - 1u)) << (a - 1 - s * R);
  }
  if (m) co[w] |= m;
}

// ---------------------------------------------------------------------------------------------
// cs219 ungapped prefilter (Prefilter::ungapped_sse_score, src/hhprefilter.cpp:214-275).
//   S(i,j) = max(0, min(255, S(i-1,j-1) + prof[x_j][i]) - offset);  score = max over all cells.
// One warp per database sequence.  The query is cut into TILES of 64*WB positions (WB <= 8, one launch per
// tile, so a query of any length works); inside a tile lane l owns the contiguous positions
// [l*2WB, (l+1)*2WB) as WB registers of two 16-bit values: register w holds position l*2WB + w in its low
// half and l*2WB + WB + w in its high half.  With that pairing the diagonal predecessor of BOTH halves of
// register w is register w-1, so the sweep needs no funnel shifts: one byte-permute per column builds the
// carry into register 0 (low half: last position of lane l-1 via one shuffle, high half: position WB-1 of
// the own lane).  The u8-saturating recurrence is exact in 16-bit integers:
//   min(S + p, 255) - offset = min(S + (p - offset), 255 - offset),  then max(., 0)
// = ONE DPX instruction per two cells, __viaddmin_s16x2_relu(S, p - offset, 255 - offset); the running
// maximum takes one __vimax3_s16x2 per two registers.  The profile (p - offset as s16x2, [state][w][lane]
// words, 28 KB per WB) sits in shared memory; the 32 lanes of a warp read 128 contiguous bytes.
// Tile t > 0 needs S of the previous tile's last position at column j-1: tile t-1 stores that byte per
// column (edge_out), tile t reads it (edge_in); the per-sequence maximum is combined across tiles in `scores`.
// Positions past the end of the query carry p = 0: their S is always < the diagonal predecessor's (or 0) and
// never changes the maximum.
// ---------------------------------------------------------------------------------------------
struct PfParams {
  int n;
  const int* L;
  const long long* off;
  const uint8_t* seq;
  const uint32_t* prof32;   // this tile's profile: [220][WB][32] words (p - offset | p - offset) as s16x2
  int offset;
  int tile, last_tile;      // tile index; 1 if no further tile follows
  const uint8_t* edge_in;   // [sum L] S(last position of tile-1, column) per sequence column (tile > 0)
  uint8_t* edge_out;        // [sum L] written when !last_tile
  int* scores;              // running maximum over the tiles launched so far
  unsigned int* counter;
};

template <int WB>   // 32-bit s16x2 registers per lane: the tile covers 64*WB query positions
__global__ void __launch_bounds__(512) k_prefilter_ungapped(const PfParams P) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint32_t* sprof = reinterpret_cast<uint32_t*>(smem_raw);   // [220][WB][32]
  for (int idx = threadIdx.x; idx < 220 * WB * 32; idx += blockDim.x) sprof[idx] = P.prof32[idx];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const uint32_t cap = (uint32_t)(255 - P.offset) * 0x00010001u;           // 255 - offset | 255 - offset
  const bool first_tile = P.tile == 0;
  for (;;) {
    int n = 0;
    if (lane == 0) n = (int)atomicAdd(P.counter, 1u);
    n = __shfl_sync(0xffffffffu, n, 0);
    if (n >= P.n) break;
    const long long o = P.off[n];
    const uint8_t* x = P.seq + o;
    const int L = P.L[n];
    uint32_t S[WB];
#pragma unroll
    for (int w = 0; w < WB; ++w) S[w] = 0;
    uint32_t smax = 0;
    for (int j0 = 0; j0 < L; j0 += 32) {
      const int xl = (j0 + lane < L) ? (int)x[j0 + lane] : 0;
      // carry into the tile at column j = S(last position of the previous tile, column j-1)
      int el = 0;
      if (!first_tile && j0 + lane >= 1 && j0 + lane <= L) el = (int)P.edge_in[o + j0 + lane - 1];
      const int cnt = min(32, L - j0);
      uint32_t eout = 0;
      for (int jj = 0; jj < cnt; ++jj) {
        const int xs = __shfl_sync(0xffffffffu, xl, jj);
        const uint32_t* prow = sprof + (size_t)xs * (WB * 32) + lane;
        uint32_t up = __shfl_up_sync(0xffffffffu, S[WB - 1], 1);
        const uint32_t ein = first_tile ? 0u : (uint32_t)__shfl_sync(0xffffffffu, el, jj);   // warp-uniform branch
        if (lane == 0) up = ein << 16;
        // register 0's diagonal inputs: low half <- high half of `up` (position l*2WB-1), high half <- low half
        // of the own last register (position l*2WB+WB-1)
        const uint32_t carry = __byte_perm(up, S[WB - 1], 0x5432);
#pragma unroll
        for (int w = WB - 1; w >= 1; --w) S[w] = __viaddmin_s16x2_relu(S[w - 1], prow[w * 32], cap);
        S[0] = __viaddmin_s16x2_relu(carry, prow[0], cap);
#pragma unroll
        for (int w = 0; w + 1 < WB; w += 2) smax = __vimax3_s16x2(smax, S[w], S[w + 1]);
        if (WB & 1) smax = __vimax3_s16x2(smax, S[WB - 1], 0u);
        if (!P.last_tile) {
          // S(last position of this tile, column j0+jj): lane 31, last register, high half; lane jj keeps it
          const uint32_t e = __shfl_sync(0xffffffffu, S[WB - 1] >> 16, 31);
          if (lane == jj) eout = e;
        }
      }
      if (!P.last_tile && lane < cnt) P.edge_out[o + j0 + lane] = (uint8_t)eout;
    }
    uint32_t m = max(smax & 0xFFFFu, smax >> 16);
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, k));
    if (lane == 0) P.scores[n] = first_tile ? (int)m : max(P.scores[n], (int)m);
  }
}

// ---------------------------------------------------------------------------------------------
// Gapped byte Smith-Waterman of prefilter stage 2 (Prefilter::swStripedByte, src/hhprefilter.cpp:70-212).
// The reference's Farrar-striped AVX2 routine has 32 byte lanes and a lazy-F loop that does not update E,
// so its score can depend on the striping (SURVEY App. D-5).  To be bit-identical we execute exactly that
// algorithm: one WARP = the 32 byte lanes of the AVX2 vector (lane k owns query positions k*W + j),
// the full-width byte shift is __shfl_up, the movemask test is __all_sync.  Stage 2 only sees the
// survivors of stage 1 (hundreds..thousands of sequences), so one byte per lane is plenty.
// ---------------------------------------------------------------------------------------------
struct SwParams {
  int n;                    // number of requested sequences
  const int* ids;           // [n] sequence ids (null = 0..n-1)
  const int* L;
  const long long* off;
  const uint8_t* seq;
  const uint8_t* prof;      // striped profile [220][W][32]: byte (k, j, lane) = position lane*W + j (bias pad)
  int W;
  int gap_open, gap_extend, bias;
  int* scores;              // [n]
  unsigned int* counter;
};

template <bool PROF_SMEM>   // false: the striped profile does not fit in shared memory (Lq > ~900) and is read from L2
__global__ void __launch_bounds__(256) k_prefilter_sw(const SwParams P) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int W = P.W;
  const uint8_t* sprof = PROF_SMEM ? smem_raw : P.prof;        // [220][W][32]
  if (PROF_SMEM) {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(P.prof);
    uint32_t* dst = reinterpret_cast<uint32_t*>(smem_raw);
    for (int idx = threadIdx.x; idx < 220 * W * 8; idx += blockDim.x) dst[idx] = src[idx];
    __syncthreads();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint8_t* Hst = smem_raw + (PROF_SMEM ? (size_t)220 * W * 32 : 0) + (size_t)warp * 3 * W * 32 + lane;   // + j*32
  uint8_t* Hld = Hst + (size_t)W * 32;
  uint8_t* E = Hld + (size_t)W * 32;
  for (;;) {
    int it = 0;
    if (lane == 0) it = (int)atomicAdd(P.counter, 1u);
    it = __shfl_sync(0xffffffffu, it, 0);
    if (it >= P.n) break;
    const int id = P.ids ? P.ids[it] : it;
    const int vmax = pf_sw_sequence(sprof, W, P.seq + P.off[id], P.L[id], Hst, Hld, E, P.gap_open, P.gap_extend,
                                    P.bias, lane);
    if (lane == 0) P.scores[it] = vmax;
    __syncwarp();
  }
}


}  // namespace hhg
