// hh-suite_b200/csrc/hhg_api.cu -- the C-ABI (include/hhg.h) over the sm_90a kernels.
// Host side: planning (length-sorted 32-target warp jobs, strip work items, memory waves),
// device memory, launches.  There is no CPU fallback: without a CUDA device every entry point fails.
#include "../../include/hhg.h"
#include "hhg_kernels.cuh"
#include "hhg_hhm.cuh"
#include "hhg_msa.cuh"
#include "hhg_crf.cuh"
#include "hhg_mac.cuh"
#include "hhg_topk.cuh"
#include "hhg_hitlist.h"
#include "hhg_stage_cache.h"

#include <dlfcn.h>
#if defined(__SSE__)
#include <xmmintrin.h>     // RCPPS: the alignment weights of the reference go through it (hhg_msa.cuh)
#endif

#include <algorithm>
#include <chrono>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <cmath>
#include <cfloat>
#include <mutex>
#include <numeric>
#include <string>
#include <thread>
#include <type_traits>
#include <unordered_set>
#include <vector>

using namespace hhg;

namespace {

thread_local std::string g_err;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

#define CK(expr)                                                                                  \
  do {                                                                                            \
    cudaError_t e__ = (expr);                                                                     \
    if (e__ != cudaSuccess)                                                                       \
      return fail(e__ == cudaErrorMemoryAllocation ? HHG_ENOMEM : HHG_ECUDA, "%s: %s (%s:%d)", #expr, \
                  cudaGetErrorString(e__), __FILE__, __LINE__);                                   \
  } while (0)

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  ~DevBuf() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  cudaError_t alloc(size_t count) {
    release();
    n = count;
    if (count == 0) return cudaSuccess;
    return cudaMalloc((void**)&p, count * sizeof(T));
  }
  cudaError_t ensure(size_t count) {
    if (count <= n && p) return cudaSuccess;
    return alloc(count);
  }
};

// strip height forced by the environment (developer / test knob), or 0 = chosen per plan (plan_strip_rows)
int strip_rows() {
  const char* e = getenv("HHG_STRIP_ROWS");
  if (e) {
    int r = atoi(e);
    if (r == 8 || r == 12 || r == 16) return r;
  }
  return 0;
}

// Runs body(k) for k in [0, n) on min(16, hardware threads) host threads: worker w takes k = w, w + hw, ... and worker 0
// is the calling thread.  body returns an error message, empty when k went fine.  The result is the first failure of
// the lowest-numbered worker that failed (k = -1 when none did).
struct HostFail {
  int k = -1;
  std::string msg;
};

template <typename F>
HostFail host_for(int n, F&& body) {
  const unsigned hw = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
  std::vector<HostFail> fails(hw);
  auto work = [&](unsigned w) {
    for (int k = (int)w; k < n; k += (int)hw) {
      std::string msg = body(k);
      if (!msg.empty() && fails[w].k < 0) fails[w] = {k, std::move(msg)};
    }
  };
  std::vector<std::thread> pool;
  for (unsigned w = 1; w < hw; ++w) pool.emplace_back(work, w);
  work(0);
  for (auto& th : pool) th.join();
  for (auto& f : fails)
    if (f.k >= 0) return f;
  return {};
}

}  // namespace

struct hhg_ctx {
  int device = 0;
  std::shared_ptr<void> msa_cache;     // MsaChunk reused by the single-alignment calls (hhg_msa_to_hmm, hhg_query_from_a3m)
  std::shared_ptr<void> crf_cache;     // device + pinned host staging of hhg_query_context_pseudocounts
  std::shared_ptr<void> msa_rcp;       // DevBuf<float>: the host's RCPPS table (hhg_msa.cuh), uploaded once per context
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  int sm_count = 0;
  long long launches = 0;
  // query
  int Lq = 0, R = 0;     // Lq: length of query 0; R: forced strip height (HHG_STRIP_ROWS) or 0 = per plan
  // query batch (hhg_query_set = a batch of one): lengths, first row record of each query in qrec, average aa
  // frequencies (for the fused null model of batch searches over a raw shard)
  int nq = 0;
  std::vector<int> q_L, q_row0;
  std::vector<float> h_q_pav;
  bool has_q_pav = false;
  DevBuf<float> d_q_pav, d_pb;
  float h_pb[20] = {};   // host copy of d_pb (the background of columnscore 0 in the last batch search)
  // excluded regions (-excl / -template_excl), applied to every search until cleared: ex = {q_lo[ex_nq], q_hi[ex_nq],
  // t_lo[ex_nt], t_hi[ex_nt]} as k_celloff_regions and k_mac_realign read it from d_ex
  std::vector<int> ex;
  int ex_nq = 0, ex_nt = 0;
  DevBuf<int> d_ex;
  unsigned long long query_serial = 0;   // bumped by every hhg_query_set*: plans built for an older batch are rebuilt
  int group_jobs = 16;   // work-item interleave (see k_viterbi): 16 jobs x nstrips items keep the group L2-resident
  uint32_t epoch = 0;    // run counter feeding the boundary-slot tags
  uint32_t epoch_window = 1;   // number of times the 20-bit epoch has wrapped (+1)
  DevBuf<float4> qrec;
  DevBuf<float> S33;
  DevBuf<float> lg2, diff;   // fast_log2 tables for Hit.score
  std::vector<float> h_lg2;
  bool has_ss = false, has_S33 = false;
  hhg_params par{1, 0.f, 0.f, -0.03f, 0.11f, 0, 0.1f, 2};
  // prefilter
  DevBuf<uint8_t> pf_prof, sw_prof;
  DevBuf<uint8_t> pf_edge[2];   // per-column hand-off between query tiles of the ungapped prefilter (Lq > 512)
  DevBuf<int> sw_ids, sw_scores;
  DevBuf<unsigned> pf_counter, pf_hist;
  DevBuf<int> pf_corr, pf_ids_a;   // corrected scores, survivor lists of the stage-1 selection
  // query-batch prefilter: raw scores [nq][n] of the last hhg_prefilter_ungapped_batch_run and the shard they cover
  DevBuf<int> pfb_scores;
  unsigned long long pfb_db_serial = 0;
  int pfb_nq = 0;
  DevBuf<PfSlab> pfb_slabs;
  DevBuf<PfCut> pfb_cuts;
  DevBuf<float> pfb_flog2;
  DevBuf<int4> swb_items;
  DevBuf<SwBatchQuery> swb_queries;
  // MAC realignment (hhg_mac_*): the query batch in linear transition space (hhg_mac_query_set = a batch of one) +
  // grow-only scratch of the last call
  int mac_nq = 0;                        // 0: no query set
  std::vector<int> mac_qL;
  bool mac_has_q_pav = false;
  DevBuf<float> mac_qp, mac_qtr, mac_q_pav, mac_pb, mac_ttr, mac_post, mac_out_post;
  DevBuf<int> mac_qL_d;
  DevBuf<long long> mac_qoff;            // [2*nq]: first float of each query's p, then of its transitions
  DevBuf<float4> mac_cols;               // template records of one memory wave, null model applied (raw shards)
  DevBuf<uint8_t> mac_off, mac_bt, mac_out_states;
  DevBuf<double> mac_rows, mac_scale;
  DevBuf<long long> mac_i64, mac_dbg;
  DevBuf<int> mac_i32, mac_out_i, mac_out_j, mac_map;
  cudaStream_t aux_stream = nullptr;     // long-template launch of hhg_mac_realign
  cudaEvent_t aux_ev[2] = {nullptr, nullptr};
  DevBuf<MacHitOut> mac_out;
  std::vector<long long> mac_cell_off;   // of the last call (debug fetch), relative to its memory wave
  std::vector<int> mac_Lt, mac_req_Lq;
  int mac_waves = 0;                     // memory waves of the last call: the posteriors stay readable after one
  size_t max_bt_bytes = 0;   // memory-wave budget for backtrace words (and for the MAC realignment's scratch)
  struct hhg_plan* scratch_plan = nullptr;   // reused by hhg_viterbi_search
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
};

static std::atomic<unsigned long long> g_db_serial{1};

// Page-locked, device-mapped host memory holding the raw records of a whole database (hhg_dbstore_*).
struct hhg_dbstore {
  int device = 0;
  bool has_ss = false;
  int cap_targets = 0, n = 0;
  long long cap_cols = 0, total_cols = 0;
  std::vector<int> L;
  std::vector<long long> col_off;
  ColRec* cols = nullptr;        // host addresses (cudaHostAlloc, mapped) ...
  float* pav = nullptr;
  const float4* d_cols = nullptr;   // ... and what the device calls them
  const float* d_pav = nullptr;
  int users = 0;                 // staged shards made over this store
};

// A database's own ffindex records as the source of a staged shard (hhg_recsrc_*): the record text stays the
// caller's (typically an mmap of the ffdata); only offsets, lengths and parameters are copied.
struct hhg_recsrc {
  int device = 0;
  int kind = 0;                     // 0 HHM, 1 A3M, 2 compressed A3M
  int n = 0;
  const char* data = nullptr;
  std::vector<int64_t> off, len;
  hhg_seqdb seqs{};                 // compressed A3M: the sequence database (its arrays stay the caller's)
  hhg_msa_params mp{};
  hhg_prep_params pp{};
  std::vector<float> S, pb, R;      // S empty: not given
  bool has_ss = false;
  std::vector<int32_t> L;           // columns of each record, 0 until a stage call has scanned it
  int users = 0;                    // staged shards made over this source
};

struct hhg_db {
  // identity for plan reuse (addresses get recycled); a staged shard takes a new one whenever hhg_db_stage changes a slot
  unsigned long long serial = g_db_serial.fetch_add(1);
  int device = 0;
  int n = 0;
  long long total_cols = 0;
  bool has_ss = false;
  std::vector<int> L;
  std::vector<long long> col_off;
  DevBuf<int> dL;
  DevBuf<long long> dcol_off;
  DevBuf<float4> cols;       // prepared column records (what the DP reads)
  bool raw = false;          // created by hhg_db_create_raw: cols is filled by hhg_db_apply_null_model
  DevBuf<float4> cols_raw;   // pre-null-model records
  DevBuf<float> pav;         // [n*20] template average aa frequencies
  bool prepared = true;
  unsigned long long cols_version = 1;   // bumped whenever `cols` is rewritten (hhg_db_apply_null_model)
  // staged shard (hhg_db_create_staged): n slots over an arena of total_cols records; L[s] == 0 marks an empty slot
  hhg_dbstore* store = nullptr;
  std::unique_ptr<StageCache> stage;
  DevBuf<StageDesc> d_desc;
  DevBuf<int> d_slot_id, d_zero;         // 0..n-1 and zeros: k_mac_gather_cols' request arrays for a pass over all slots
  // record-sourced staged shard (hhg_db_create_staged_records): targets are built from src's records
  hhg_recsrc* src = nullptr;
  std::shared_ptr<void> builder;         // the source's MsaBuilder / HhmBuilder, device buffers kept between calls
  std::vector<float> neff;               // [n] Neff_HMM of the target in each slot
  DevBuf<float4> rec_cols;               // one group's built records and pav rows: k_stage_gather's source
  DevBuf<float> rec_pav;
};

struct hhg_csdb {
  const unsigned long long serial = g_db_serial.fetch_add(1);   // identity of the shard the batch scores cover
  int device = 0;
  int n = 0;
  long long total = 0;
  DevBuf<int> dL;
  DevBuf<long long> doff;
  DevBuf<uint8_t> seq;
  DevBuf<int> scores;
};

struct Wave {
  int job_begin = 0, job_end = 0;
  long long item_begin = 0, item_end = 0;   // slice of the plan's work-item table (job index relative to job_begin)
};

struct hhg_plan {
  bool built = false;   // false after a failed (re)build: the host tables no longer describe the device buffers
  const hhg_db* db = nullptr;
  unsigned long long db_serial = 0;
  int device = 0;
  int n = 0;            // requests
  int Lq = 0, R = 16;   // Lq: length of query 0 (single-query callers)
  std::vector<int> q_L, q_row0;          // query batch geometry the plan was built for
  std::vector<int> req_query;            // request -> query index
  int njobs = 0;
  long long ss_total = 0, co_total = 0;  // per-strip maxima blocks / cell-off words over all jobs
  double cells = 0, padded_cells = 0, alg_bytes = 0;
  std::vector<int> ids;          // request -> target id
  std::vector<int> order;        // sorted position -> request index
  std::vector<JobDesc> jobs;     // [njobs]
  std::vector<ReqDesc> reqs;     // [n] in request order
  std::vector<int2> items;
  long long jc_total = 0;                 // float4 in the job-interleaved operand stream
  unsigned long long jc_version = 0;      // db->cols_version the stream was built from (0 = never)
  int nm_mode = -1;                       // >= 0: columnscore of the null model fused into the stream (raw shard)
  int jc_nm_mode = -2;                    // nm_mode / query batch the stream was built with
  unsigned long long jc_query_serial = 0;
  float jc_pb[20] = {};                   // pb the stream was divided by (nm_mode 0)
  std::vector<Wave> waves;
  long long path_total = 0;
  // device
  DevBuf<JobDesc> d_jobs;
  DevBuf<ReqDesc> d_reqs;
  DevBuf<int> d_job_target;
  DevBuf<int2> d_items;
  DevBuf<float> d_S;
  DevBuf<float4> d_jcols;
  DevBuf<uint32_t> d_bt, d_co;
  DevBuf<BndSlot> d_bnd;
  uint32_t bnd_epoch_window = 0;   // epoch window in which d_bnd was last cleared
  DevBuf<float> d_strip_score;
  DevBuf<int> d_strip_ij;
  DevBuf<unsigned> d_counter;
  float ms_viterbi = 0, ms_backtrace = 0;   // filled by hhg_plan_run_timed
  size_t max_bt_bytes = 0;
  DevBuf<uint8_t> d_paths_compact;
  DevBuf<long long> d_compact_off;
  std::vector<long long> h_compact_off;
  DevBuf<HitRec> d_hits;
  // top-K selection / exchange scratch (hhg_plan_topk)
  DevBuf<unsigned long long> d_keys;
  DevBuf<int> d_gids;
  DevBuf<float> d_user_key;
  DevBuf<TopkState> d_topk_state;
  DevBuf<TopkRec> d_topk_local, d_topk_all;
  DevBuf<uint8_t> d_topk_paths;
  DevBuf<uint8_t> d_paths;
  // cell-off input (optional)
  bool celloff = false;
  int n_excl_steps = 0;
  DevBuf<int> d_step_req, d_step_i, d_step_j;
};

const char* hhg_last_error(void) { return g_err.c_str(); }

int hhg_ctx_create(int device, void* stream, hhg_ctx** out) {
  if (!out) return fail(HHG_EINVAL, "out is NULL");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(HHG_ENODEV, "no CUDA device available (%s); this library has no CPU fallback",
                cudaGetErrorString(e));
  if (device < 0) CK(cudaGetDevice(&device));
  if (device >= ndev) return fail(HHG_EINVAL, "device %d out of range (%d devices)", device, ndev);
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  // sm_90a code only loads on compute capability 9.0 (H100)
  if (prop.major != 9 || prop.minor != 0)
    return fail(HHG_ENODEV, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device,
                prop.major, prop.minor);
  std::unique_ptr<hhg_ctx> holder(new hhg_ctx());
  hhg_ctx* c = holder.get();
  c->device = device;
  c->sm_count = prop.multiProcessorCount;
  if (stream) {
    c->stream = (cudaStream_t)stream;
  } else {
    CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    c->own_stream = true;
  }
  c->R = strip_rows();
  {
    // fast_log2 tables exactly as the reference fills them on first use (src/util-inl.h:113-121):
    // lg2[i] = log2(1 + i/1024) via the C library's double-precision log (that is the overload the
    // reference's expression resolves to; verified against its table), diff[i] = slope / 8096
    std::vector<float> lg2(1025, 0.f), diff(1025, 0.f);
    float prev = 0.0f;
    for (int i = 1; i <= 1024; ++i) {
      lg2[i] = (float)(::log((double)(1024 + i)) * 1.442695041 - 10.0);
      diff[i - 1] = (float)((double)(lg2[i] - prev) * 1.2352E-4);
      prev = lg2[i];
    }
    c->h_lg2 = lg2;
    cudaError_t e1 = c->lg2.alloc(1025), e2 = c->diff.alloc(1025);
    if (e1 != cudaSuccess || e2 != cudaSuccess) return fail(HHG_ENOMEM, "fast_log2 tables");
    CK(cudaMemcpy(c->lg2.p, lg2.data(), 1025 * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(c->diff.p, diff.data(), 1025 * 4, cudaMemcpyHostToDevice));
  }
  { const char* ge = getenv("HHG_GROUP_JOBS"); c->group_jobs = ge ? std::max(1, atoi(ge)) : 16; }
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const char* env = getenv("HHG_MAX_BT_GB");
  double cap = env ? atof(env) * 1e9 : 48e9;
  c->max_bt_bytes = (size_t)std::min(cap, 0.45 * (double)free_b);
  *out = holder.release();
  return HHG_OK;
}

int hhg_ctx_destroy(hhg_ctx* ctx) {
  if (!ctx) return HHG_OK;
  cudaSetDevice(ctx->device);
  if (ctx->scratch_plan) hhg_plan_destroy(ctx->scratch_plan);
  for (auto& e : ctx->ev) if (e) cudaEventDestroy(e);
  for (auto& e : ctx->aux_ev) if (e) cudaEventDestroy(e);
  if (ctx->aux_stream) cudaStreamDestroy(ctx->aux_stream);
  if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
  return HHG_OK;
}

int hhg_ctx_sync(hhg_ctx* ctx) {
  if (!ctx) return fail(HHG_EINVAL, "ctx is NULL");
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

long long hhg_ctx_launch_count(hhg_ctx* ctx) { return ctx ? ctx->launches : 0; }

// The context's second stream and its two events, made on first use (long-template MAC launch, hhg_db_stage).
static int ctx_aux_stream(hhg_ctx* ctx) {
  if (ctx->aux_stream) return HHG_OK;
  CK(cudaStreamCreateWithFlags(&ctx->aux_stream, cudaStreamNonBlocking));
  CK(cudaEventCreateWithFlags(&ctx->aux_ev[0], cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&ctx->aux_ev[1], cudaEventDisableTiming));
  return HHG_OK;
}

// ------------------------------------------------------------------------------------------ DB
static int pack_profiles(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* p_off,
                         const int64_t* tr_off, const int64_t* ss_off, const float* p, const float* tr,
                         const uint8_t* ss, const std::vector<long long>& col_off, long long total_cols,
                         float4* d_out) {
  // upload the raw profiles in bounded chunks of targets, pack on the device
  const size_t kChunkBytes = (size_t)1 << 30;
  DevBuf<float> dp, dtr;
  DevBuf<uint8_t> dss;
  DevBuf<int> dL;
  DevBuf<long long> dcol, dpo, dto, dso;
  int t0 = 0;
  while (t0 < n) {
    // the profiles of consecutive targets need not be contiguous in the caller's arrays; upload per
    // target range [lo, hi) covering min..max offsets when contiguous, else target by target.
    int t1 = t0;
    size_t bytes = 0;
    while (t1 < n && (bytes == 0 || bytes + (size_t)(L[t1] + 2) * 80 < kChunkBytes)) {
      bytes += (size_t)(L[t1] + 2) * 80;
      ++t1;
    }
    const int m = t1 - t0;
    std::vector<long long> po(m), to(m), so(m), co(m);
    std::vector<int> LL(m);
    size_t np = 0, ntr = 0, nss = 0;
    for (int k = 0; k < m; ++k) {
      LL[k] = L[t0 + k];
      po[k] = (long long)np; to[k] = (long long)ntr; so[k] = (long long)nss;
      co[k] = col_off[t0 + k] - col_off[t0];
      np += (size_t)(LL[k] + 2) * 20; ntr += (size_t)(LL[k] + 1) * 7; nss += (size_t)(LL[k] + 2);
    }
    std::vector<float> hp(np), htr(ntr);
    std::vector<uint8_t> hss(ss ? nss : 0);
    for (int k = 0; k < m; ++k) {
      memcpy(hp.data() + po[k], p + p_off[t0 + k], (size_t)(LL[k] + 2) * 20 * sizeof(float));
      memcpy(htr.data() + to[k], tr + tr_off[t0 + k], (size_t)(LL[k] + 1) * 7 * sizeof(float));
      if (ss) memcpy(hss.data() + so[k], ss + ss_off[t0 + k], (size_t)(LL[k] + 2));
    }
    const long long cols = (t1 < n ? col_off[t1] : total_cols) - col_off[t0];
    CK(dp.ensure(np)); CK(dtr.ensure(ntr)); CK(dL.ensure(m)); CK(dcol.ensure(m)); CK(dpo.ensure(m));
    CK(dto.ensure(m)); CK(dso.ensure(m));
    if (ss) CK(dss.ensure(nss));
    CK(cudaMemcpyAsync(dp.p, hp.data(), np * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(dtr.p, htr.data(), ntr * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (ss) CK(cudaMemcpyAsync(dss.p, hss.data(), nss, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(dL.p, LL.data(), m * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(dcol.p, co.data(), m * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(dpo.p, po.data(), m * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(dto.p, to.data(), m * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(dso.p, so.data(), m * 8, cudaMemcpyHostToDevice, ctx->stream));
    const int threads = 128;
    const long long blocks = (cols + threads - 1) / threads;
    k_pack_cols<<<(unsigned)blocks, threads, 0, ctx->stream>>>(
        m, dL.p, dcol.p, dpo.p, dto.p, dso.p, dp.p, dtr.p, ss ? dss.p : nullptr,
        reinterpret_cast<ColRec*>(d_out) + col_off[t0], cols);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ctx->stream));   // host staging vectors die at scope end
    t0 = t1;
  }
  return HHG_OK;
}

// A new shard of n entries with lengths L, each in [1, 32767] (`what` names an entry in the error: "target" or
// "record"): column offsets, device buffers (cols; cols_raw and pav too for a raw shard), L and col_off uploaded.
static int db_new(hhg_ctx* ctx, int n, const int32_t* L, bool raw, const char* what, std::unique_ptr<hhg_db>* out) {
  std::unique_ptr<hhg_db> db(new hhg_db());
  db->device = ctx->device;
  db->n = n;
  db->L.assign(L, L + n);
  db->col_off.resize(n);
  long long tot = 0;
  for (int k = 0; k < n; ++k) {
    if (L[k] < 1 || L[k] > 32767) return fail(HHG_EINVAL, "%s %d: length %d out of [1,32767]", what, k, L[k]);
    db->col_off[k] = tot;
    tot += L[k];
  }
  db->total_cols = tot;
  CK(db->cols.alloc((size_t)tot * 7));
  if (raw) CK(db->cols_raw.alloc((size_t)tot * 7));
  CK(db->dL.alloc(n));
  CK(db->dcol_off.alloc(n));
  if (raw) CK(db->pav.alloc((size_t)n * 20));
  CK(cudaMemcpyAsync(db->dL.p, db->L.data(), (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(db->dcol_off.p, db->col_off.data(), (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  *out = std::move(db);
  return HHG_OK;
}

// A raw shard whose cols_raw and pav are written (or queued on ctx->stream): cols starts as a copy of cols_raw and is
// rewritten by hhg_db_apply_null_model.
static int db_publish_raw(hhg_ctx* ctx, std::unique_ptr<hhg_db>& holder, hhg_db** out) {
  hhg_db* db = holder.get();
  CK(cudaMemcpyAsync(db->cols.p, db->cols_raw.p, db->cols.n * sizeof(float4), cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  db->raw = true;
  db->prepared = false;
  *out = holder.release();
  return HHG_OK;
}

// pav == NULL: a prepared shard (hhg_db_create), else a raw one (hhg_db_create_raw)
static int db_create_impl(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* p_off, const int64_t* tr_off,
                          const int64_t* ss_off, const float* p, const float* tr, const uint8_t* ss, const float* pav,
                          hhg_db** out) {
  if (!ctx || !out || n <= 0 || !L || !p_off || !tr_off || !p || !tr)
    return fail(HHG_EINVAL, "hhg_db_create: bad argument");
  if (ss && !ss_off) return fail(HHG_EINVAL, "hhg_db_create: ss given without ss_off");
  CK(cudaSetDevice(ctx->device));
  std::unique_ptr<hhg_db> holder;   // freed on every early return below
  int rc = db_new(ctx, n, L, pav != nullptr, "target", &holder);
  if (rc != HHG_OK) return rc;
  hhg_db* db = holder.get();
  db->has_ss = ss != nullptr;
  rc = pack_profiles(ctx, n, L, p_off, tr_off, ss_off, p, tr, ss, db->col_off, db->total_cols,
                     pav ? db->cols_raw.p : db->cols.p);
  if (rc != HHG_OK) return rc;
  if (pav) {
    CK(cudaMemcpyAsync(db->pav.p, pav, (size_t)n * 20 * 4, cudaMemcpyHostToDevice, ctx->stream));
    return db_publish_raw(ctx, holder, out);
  }
  CK(cudaStreamSynchronize(ctx->stream));
  *out = holder.release();
  return HHG_OK;
}

int hhg_db_create(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* p_off, const int64_t* tr_off,
                  const int64_t* ss_off, const float* p, const float* tr, const uint8_t* ss,
                  hhg_db** out) {
  return db_create_impl(ctx, n, L, p_off, tr_off, ss_off, p, tr, ss, nullptr, out);
}

int hhg_db_create_raw(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* p_off, const int64_t* tr_off,
                      const int64_t* ss_off, const float* p, const float* tr, const uint8_t* ss,
                      const float* pav, hhg_db** out) {
  if (!pav) return fail(HHG_EINVAL, "hhg_db_create_raw: pav is NULL");
  return db_create_impl(ctx, n, L, p_off, tr_off, ss_off, p, tr, ss, pav, out);
}

int hhg_db_apply_null_model(hhg_ctx* ctx, hhg_db* db, const float* q_pav, const float* pb, int columnscore) {
  if (!ctx || !db || !db->raw) return fail(HHG_EINVAL, "hhg_db_apply_null_model: db was not created raw");
  if (columnscore < 0 || columnscore > 3) return fail(HHG_EINVAL, "columnscore %d not supported (0..3)", columnscore);
  if ((columnscore == 1 || columnscore == 3) && !q_pav) return fail(HHG_EINVAL, "q_pav is NULL");
  if (columnscore == 0 && !pb) return fail(HHG_EINVAL, "pb is NULL");
  CK(cudaSetDevice(ctx->device));
  DevBuf<float> dq;
  CK(dq.alloc(40));
  float h[40] = {0};
  if (q_pav) memcpy(h, q_pav, 80);
  if (pb) memcpy(h + 20, pb, 80);
  CK(cudaMemcpyAsync(dq.p, h, 160, cudaMemcpyHostToDevice, ctx->stream));
  if (db->stage) {
    // arena runs are in no order, so k_null_model's bisection over col_off does not apply: one k_mac_gather_cols
    // "request" per slot with query 0 copies the slot's records in place of the arena (empty slots have L = 0)
    for (int s0 = 0; s0 < db->n; s0 += 65535) {
      const int k = std::min(db->n - s0, 65535);
      k_mac_gather_cols<<<dim3(4, k), 128, 0, ctx->stream>>>(k, db->d_zero.p, db->d_slot_id.p + s0, db->dL.p + s0,
                                                             db->dcol_off.p, db->dcol_off.p + s0, db->cols_raw.p, db->pav.p,
                                                             dq.p, dq.p + 20, columnscore, db->cols.p);
      ctx->launches++;
    }
  } else {
    const int threads = 128;
    k_null_model<<<(unsigned)((db->total_cols + threads - 1) / threads), threads, 0, ctx->stream>>>(
        db->total_cols, db->n, db->dcol_off.p, db->cols_raw.p, db->pav.p, dq.p, dq.p + 20, columnscore,
        db->cols.p);
    ctx->launches++;
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->stream));
  db->prepared = true;
  db->cols_version++;
  return HHG_OK;
}

// ------------------------------------------------------------------------------ DB from HHM text records
// HHEntry::getTemplateHMM + the query-independent part of PrepareTemplateHMM, once per database load.
// ---------------------------------------------------------------------------------------------------------------
// A3M alignments -> HMMs (hhg_msa.cuh).  One chunk of parsed alignments goes through filter, weights, M state and
// finish; the callers either export the raw HMM (hhg_msa_to_hmm) or continue into the pseudocount step and the shard.
namespace {

struct MsaChunk {
  std::vector<MsaHost> host;
  std::vector<MsaDesc> desc;
  long long seq_total = 0, col_total = 0, x_total = 0, ins_total = 0;
  int Lmax = 0, Nmax = 0;
  DevBuf<MsaDesc> d_desc;
  DevBuf<uint8_t> X, member;
  DevBuf<int8_t> keep, display;
  DevBuf<int> first, last, nres, ksort, in_, inkk, seqid_prev, acc, Ncnt, Nmaxv, idw, ins_k, nfil, status, ni, counter, cnt;
  DevBuf<uint16_t> ins_cnt;
  DevBuf<uint32_t> ins_off;
  DevBuf<float> wg, f, tr, nm, ni_f, nd, nseg, nhmm, wc, wi, pb;
  DevBuf<long long> item_off;
  MsaArrays A{};
};

const float* msa_rcp_table(hhg_ctx* ctx) {
  // RCPPS of this host for every integer argument the weighting can produce (src/hhalignment.cpp:2531)
  static std::vector<float> table;
  static std::once_flag once;
  std::call_once(once, [] {
    table.resize(MSA_RCP_N);
#if defined(__SSE__)
    for (int m = 0; m < MSA_RCP_N; m += 4) {
      const __m128 v = _mm_set_ps((float)(m + 3), (float)(m + 2), (float)(m + 1), (float)m);
      _mm_storeu_ps(&table[m], _mm_rcp_ps(v));
    }
#else
    // no RCPPS on this host: the reference is built through SIMDe there, whose reciprocal estimate differs again;
    // the exact quotient keeps the result well defined (it will not be bit-identical to such a reference build)
    for (int m = 0; m < MSA_RCP_N; ++m) table[m] = 1.0f / (float)m;
#endif
  });
  if (!ctx->msa_rcp) {
    auto buf = std::make_shared<DevBuf<float>>();
    if (buf->alloc(MSA_RCP_N) != cudaSuccess) return nullptr;
    if (cudaMemcpyAsync(buf->p, table.data(), (size_t)MSA_RCP_N * 4, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) return nullptr;
    ctx->msa_rcp = buf;
  }
  return std::static_pointer_cast<DevBuf<float>>(ctx->msa_rcp)->p;
}

template <typename T, typename V>
int msa_upload(hhg_ctx* ctx, DevBuf<T>& d, const std::vector<V>& h) {
  static_assert(sizeof(T) == sizeof(V), "element size");
  CK(d.ensure(h.size() ? h.size() : 1));
  if (!h.empty()) CK(cudaMemcpyAsync(d.p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  return HHG_OK;
}

// C.host is filled (parsed); runs the four kernels and leaves f / tr / Neff / keep / wg on the device.  An error names
// alignment k by rec[k] (rec NULL: by k).
int msa_chunk_run(hhg_ctx* ctx, MsaChunk& C, const hhg_msa_params& mp, const float* S, const float* pb, const int32_t* rec) {
  const int m = (int)C.host.size();
  C.desc.resize(m);
  C.seq_total = C.col_total = C.x_total = C.ins_total = 0;
  C.Lmax = C.Nmax = 0;
  std::vector<long long> item_off(m);
  long long items = 0;
  for (int k = 0; k < m; ++k) {
    const MsaHost& H = C.host[k];
    MsaDesc& d = C.desc[k];
    d.N = H.N_in; d.L = H.L; d.stride = H.stride; d.kfirst = H.kfirst;
    d.x_off = C.x_total; d.seq_off = C.seq_total; d.col_off = C.col_total; d.ins_base = C.ins_total;
    C.x_total += (long long)H.N_in * H.stride;
    C.seq_total += H.N_in;
    C.col_total += H.L + 2;
    C.ins_total += (long long)H.ins_k.size();
    C.Lmax = std::max(C.Lmax, H.L); C.Nmax = std::max(C.Nmax, H.N_in);
    item_off[k] = items;
    items += H.L;
  }
  std::vector<uint8_t> X((size_t)C.x_total);
  std::vector<int8_t> keep((size_t)C.seq_total), display((size_t)C.seq_total);
  std::vector<int> first((size_t)C.seq_total), last((size_t)C.seq_total), nres((size_t)C.seq_total), ksort((size_t)C.seq_total);
  std::vector<uint32_t> ins_off((size_t)C.col_total);
  std::vector<int> ins_k((size_t)C.ins_total);
  std::vector<uint16_t> ins_cnt((size_t)C.ins_total);
  for (int k = 0; k < m; ++k) {
    const MsaHost& H = C.host[k];
    const MsaDesc& d = C.desc[k];
    memcpy(X.data() + d.x_off, H.X.data(), H.X.size());
    memcpy(keep.data() + d.seq_off, H.keep.data(), H.N_in);
    memcpy(display.data() + d.seq_off, H.display.data(), H.N_in);
    memcpy(first.data() + d.seq_off, H.first.data(), (size_t)H.N_in * 4);
    memcpy(last.data() + d.seq_off, H.last.data(), (size_t)H.N_in * 4);
    memcpy(nres.data() + d.seq_off, H.nres.data(), (size_t)H.N_in * 4);
    memcpy(ksort.data() + d.seq_off, H.ksort.data(), (size_t)H.N_in * 4);
    memcpy(ins_off.data() + d.col_off, H.ins_off.data(), (size_t)(H.L + 2) * 4);
    if (!H.ins_k.empty()) {
      memcpy(ins_k.data() + d.ins_base, H.ins_k.data(), H.ins_k.size() * 4);
      memcpy(ins_cnt.data() + d.ins_base, H.ins_cnt.data(), H.ins_cnt.size() * 2);
    }
  }
  int rc;
  if ((rc = msa_upload(ctx, C.d_desc, C.desc)) || (rc = msa_upload(ctx, C.X, X)) || (rc = msa_upload(ctx, C.keep, keep)) ||
      (rc = msa_upload(ctx, C.display, display)) || (rc = msa_upload(ctx, C.first, first)) || (rc = msa_upload(ctx, C.last, last)) ||
      (rc = msa_upload(ctx, C.nres, nres)) || (rc = msa_upload(ctx, C.ksort, ksort)) || (rc = msa_upload(ctx, C.ins_off, ins_off)) ||
      (rc = msa_upload(ctx, C.ins_k, ins_k)) || (rc = msa_upload(ctx, C.ins_cnt, ins_cnt)) || (rc = msa_upload(ctx, C.item_off, item_off)))
    return rc;
  const size_t ns = (size_t)C.seq_total, nc = (size_t)C.col_total;
  CK(C.in_.ensure(ns)); CK(C.inkk.ensure(ns)); CK(C.seqid_prev.ensure(ns)); CK(C.acc.ensure(ns)); CK(C.wg.ensure(ns));
  CK(C.Ncnt.ensure(nc)); CK(C.Nmaxv.ensure(nc)); CK(C.idw.ensure(nc)); CK(C.ni.ensure(nc * 21));
  CK(C.f.ensure(nc * 20)); CK(C.tr.ensure(nc * 7)); CK(C.nm.ensure(nc)); CK(C.ni_f.ensure(nc)); CK(C.nd.ensure(nc));
  CK(C.nseg.ensure(nc)); CK(C.nhmm.ensure(m)); CK(C.nfil.ensure(m)); CK(C.status.ensure(m)); CK(C.counter.ensure(1));
  CK(C.pb.ensure(20));
  CK(cudaMemcpyAsync(C.pb.p, pb, 80, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(C.status.p, 0, (size_t)m * 4, ctx->stream));
  CK(cudaMemsetAsync(C.counter.p, 0, 4, ctx->stream));
  CK(cudaMemsetAsync(C.nseg.p, 0, nc * 4, ctx->stream));
  CK(cudaMemsetAsync(C.tr.p, 0, nc * 7 * 4, ctx->stream));
  const float* rcp = msa_rcp_table(ctx);
  if (!rcp) return fail(HHG_ECUDA, "reciprocal table upload failed");
  const int sms = ctx->sm_count;
  // k_msa_mstate is latency bound inside a block (ordered sums, barriers): 12 blocks of 128 threads per SM = its register /
  // shared-memory residency (40 registers, 16 KB), every block pulls (alignment, column) items until the queue is empty
  const int nblk = (int)std::min<long long>((long long)sms * 12, std::max<long long>(items, 1));
  CK(C.cnt.ensure((size_t)nblk * (C.Lmax + 2) * 24)); CK(C.wc.ensure((size_t)nblk * (C.Lmax + 2) * 24));
  CK(C.wi.ensure((size_t)nblk * C.Nmax)); CK(C.member.ensure((size_t)nblk * C.Nmax));

  MsaArrays& A = C.A;
  A.desc = C.d_desc.p; A.X = C.X.p; A.keep = C.keep.p; A.display = C.display.p;
  A.first = C.first.p; A.last = C.last.p; A.nres = C.nres.p; A.ksort = C.ksort.p;
  A.in_ = C.in_.p; A.inkk = C.inkk.p; A.seqid_prev = C.seqid_prev.p; A.acc = C.acc.p;
  A.Ncnt = C.Ncnt.p; A.Nmax = C.Nmaxv.p; A.idmaxwin = C.idw.p; A.wg = C.wg.p;
  A.ins_off = C.ins_off.p; A.ins_k = C.ins_k.p; A.ins_cnt = C.ins_cnt.p;
  A.n_filtered = C.nfil.p; A.status = C.status.p;
  A.f = C.f.p; A.tr = C.tr.p; A.neff_m = C.nm.p; A.neff_i = C.ni_f.p; A.neff_d = C.nd.p; A.neff_seg = C.nseg.p; A.neff_hmm = C.nhmm.p;

  MsaFilterParams FP;
  FP.max_seqid = mp.max_seqid; FP.coverage = mp.coverage; FP.qid = mp.qid; FP.Ndiff = mp.Ndiff; FP.qsc = mp.qsc;
  if (S) memcpy(FP.S, S, sizeof(FP.S)); else memset(FP.S, 0, sizeof(FP.S));
  const bool timing = getenv("HHG_TIMING") != nullptr;
  cudaEvent_t ev[5] = {};
  if (timing) for (auto& e : ev) cudaEventCreate(&e);
  if (timing) cudaEventRecord(ev[0], ctx->stream);
  k_msa_filter<<<m, 256, 0, ctx->stream>>>(A, FP);
  if (timing) cudaEventRecord(ev[1], ctx->stream);
  k_msa_weights<<<m, 256, 0, ctx->stream>>>(A, C.ni.p);
  if (timing) cudaEventRecord(ev[2], ctx->stream);
  k_msa_mstate<<<nblk, MSA_MSTATE_THREADS, 0, ctx->stream>>>(A, m, C.item_off.p, items, C.counter.p, C.cnt.p, C.wc.p, C.wi.p, C.member.p,
                                              C.Lmax, C.Nmax, rcp, C.pb.p, mp.wg ? 1 : 0, ctx->lg2.p, ctx->diff.p);
  if (timing) cudaEventRecord(ev[3], ctx->stream);
  k_msa_finish<<<m, 256, 0, ctx->stream>>>(A, C.pb.p, mp.wg ? 1 : 0, ctx->lg2.p, ctx->diff.p);
  if (timing) cudaEventRecord(ev[4], ctx->stream);
  ctx->launches += 4;
  CK(cudaGetLastError());
  if (timing) {
    cudaEventSynchronize(ev[4]);
    float t[4];
    for (int k = 0; k < 4; ++k) cudaEventElapsedTime(&t[k], ev[k], ev[k + 1]);
    fprintf(stderr, "[hhg] alignment kernels (%d alignments, %lld columns): filter %.2f ms, weights %.2f ms, M state %.2f ms, finish %.2f ms\n",
            m, items, t[0], t[1], t[2], t[3]);
    for (auto& e : ev) cudaEventDestroy(e);
  }
  std::vector<int> status(m);
  CK(cudaMemcpyAsync(status.data(), C.status.p, (size_t)m * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int k = 0; k < m; ++k)
    if (status[k])
      return fail(HHG_EINVAL, "alignment %d: %s", rec ? rec[k] : k,
                  status[k] == 1 ? "contains no sequences after filtering (the reference exits here)"
                  : status[k] == 2 ? "the position-dependent identity schedule divides by zero (as in the reference)"
                                   : "no sequence left for the profile");
  return HHG_OK;
}

int msa_params_check(const hhg_msa_params* mp) {
  if (!mp) return fail(HHG_EINVAL, "alignment parameters are NULL");
  if (mp->maxseq < 2 || mp->maxseq > 65535) return fail(HHG_EINVAL, "maxseq %d outside [2, 65535]", mp->maxseq);
  if (mp->maxres < 8 || mp->maxcol < mp->maxres) return fail(HHG_EINVAL, "maxres %d / maxcol %d", mp->maxres, mp->maxcol);
  if (mp->M < 1 || mp->M > 3) return fail(HHG_EINVAL, "match-state assignment %d: 1 (A2M/A3M: upper case = match), 2 (gap percentage, Mgaps) or 3 (first sequence)", mp->M);
  if (mp->M == 2 && (mp->Mgaps < 0 || mp->Mgaps > 100)) return fail(HHG_EINVAL, "Mgaps %d outside [0, 100]", mp->Mgaps);
  if (mp->mark != 0) return fail(HHG_EINVAL, "the -mark option is not built");
  return HHG_OK;
}

// ss byte of column j (1..L) the DP reads: ss_pred * MAXCF + ss_conf (src/hhhmmsimd.cpp:133); ss_conf = 5 without an
// ss_conf row (FrequenciesAndTransitions :2313-2319)
void msa_ss_bytes(const MsaHost& H, uint8_t* out) {
  if (H.kss_pred < 0) { memset(out, 0, (size_t)H.L); return; }
  const uint8_t* pr = H.X.data() + (size_t)H.kss_pred * H.stride;
  const uint8_t* cf = H.kss_conf >= 0 ? H.X.data() + (size_t)H.kss_conf * H.stride : nullptr;
  for (int j = 1; j <= H.L; ++j) out[j - 1] = (uint8_t)((pr[j] & 0x7f) * 11 + (cf ? (cf[j] & 0x7f) : 5));
}

int seqdb_check(const hhg_seqdb* sq) {
  if (!sq) return HHG_OK;
  if (sq->n <= 0 || !sq->data || !sq->off || !sq->len) return fail(HHG_EINVAL, "sequence database: bad argument");
  return HHG_OK;
}

std::string msa_parse_any(const char* rec, int64_t len, const hhg_seqdb* sq, const hhg_msa_params* mp, MsaHost* H) {
  if (!sq) return MsaScanner::parse(rec, len, mp->maxseq, mp->maxcol, mp->maxres, H, mp->M, mp->Mgaps);
  const MsaScanner::SeqDb db{sq->n, sq->data, sq->off, sq->len};
  return MsaScanner::parse_ca3m(rec, len, db, mp->maxseq, mp->maxcol, mp->maxres, H, mp->M, mp->Mgaps);
}

// The parameter and sequence-database checks, then the parse of one alignment record (sq != NULL: compressed A3M);
// `who` prefixes a parse error.
int msa_parse_checked(const char* who, const char* rec, int64_t len, const hhg_seqdb* sq, const hhg_msa_params* mp,
                      MsaHost* H) {
  int rc = msa_params_check(mp);
  if (rc == HHG_OK) rc = seqdb_check(sq);
  if (rc != HHG_OK) return rc;
  const std::string msg = msa_parse_any(rec, len, sq, mp, H);
  if (!msg.empty()) return fail(HHG_EINVAL, "%s: %s", who, msg.c_str());
  return HHG_OK;
}

// dims[0..5] of hhg_a3m_parse / hhg_msa_to_hmm: L, N_in, N_filtered (filled in later, if at all), kfirst, kss_pred, kss_conf
void msa_dims(const MsaHost& H, int32_t* dims) {
  dims[0] = H.L; dims[1] = H.N_in; dims[2] = 0; dims[3] = H.kfirst; dims[4] = H.kss_pred; dims[5] = H.kss_conf;
}

// The template-preparation constants of hhg_prep_params and the pseudocount matrix R (src/hhhmm.cpp:1745-1752, same
// types); `who` prefixes the error of a pseudocount mode outside 0..3 (src/hhhmm.cpp:1885-1918).
int hhm_prep_args(const char* who, const hhg_prep_params* pp, const float* R, HhmPrepArgs* A) {
  if (pp->pcm < 0 || pp->pcm > 3) return fail(HHG_EINVAL, "%s: pseudocount mode %d does not exist (0..3)", who, pp->pcm);
  memcpy(A->R, R, sizeof(A->R));
  A->gapb = pp->gapb; A->gapf = pp->gapf; A->gapg = pp->gapg; A->gaph = pp->gaph; A->gapi = pp->gapi;
  A->pM2D = A->pM2I = (float)(pp->gapd * 0.0286);
  A->pM2M = 1 - A->pM2D - A->pM2I;
  A->pI2I = (float)(1.0 * pp->gape / (pp->gape - 1 + 1.0 / 0.75));
  A->pI2M = 1 - A->pI2I;
  A->pD2D = (float)(1.0 * pp->gape / (pp->gape - 1 + 1.0 / 0.75));
  A->pD2M = 1 - A->pD2D;
  A->pcm = pp->pcm; A->pca = pp->pca; A->pcb = pp->pcb; A->pcc = pp->pcc;
  return HHG_OK;
}

// AddAminoAcidPseudocounts mode 2 with pcc != 1 (src/hhhmm.cpp:1905-1909): tau = fmin(1.0, pca / (1. + pow(Neff_M/pcb, pcc)))
// with float arguments, i.e. the C library's powf, so the loaders compute it per column on the host
inline float column_tau(const hhg_prep_params* pp, float nM) {
  return (float)fmin(1.0, pp->pca / (1. + powf(nM / pp->pcb, pp->pcc)));
}

// p / tr / ss / pav of a one-record raw shard of length L as the query arrays of hhg_query_set: p[0] = p[L+1] = pav
// (CalculateAminoAcidBackground, src/hhhmm.cpp:1866), ss[0] = ss[L+1] = 0
int query_from_shard(hhg_ctx* ctx, const hhg_db* db, int L, const float* d_tr, float* p, float* tr, uint8_t* ss,
                     float* pav) {
  std::vector<ColRec> cols((size_t)L);
  CK(cudaMemcpyAsync(cols.data(), db->cols_raw.p, (size_t)L * sizeof(ColRec), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(tr, d_tr, (size_t)(L + 1) * 28, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(pav, db->pav.p, 80, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int i = 1; i <= L; ++i) {
    memcpy(p + (size_t)i * 20, cols[i - 1].p, 80);
    if (ss) ss[i] = (uint8_t)cols[i - 1].ss;
  }
  memcpy(p, pav, 80);
  memcpy(p + (size_t)(L + 1) * 20, pav, 80);
  if (ss) ss[0] = ss[L + 1] = 0;
  return HHG_OK;
}

}  // namespace

void hhg_msa_params_default(hhg_msa_params* mp) {
  if (!mp) return;
  mp->maxseq = 65535; mp->maxcol = 32765; mp->maxres = 20001;       // src/hhdecl.cpp:10-14
  mp->M = 1; mp->mark = 0;
  mp->max_seqid = 90; mp->coverage = 0; mp->qid = 0; mp->Ndiff = 100; mp->qsc = -20.0f;   // :35-39, :131-135
  mp->wg = 0;
  mp->Mgaps = 50;                                                    // :46
}

int hhg_a3m_scan(const char* rec, int64_t len, const hhg_msa_params* mp, int32_t* L, int32_t* N_in, int32_t* has_ss) {
  if (!rec || len <= 0 || !L || !N_in) return fail(HHG_EINVAL, "hhg_a3m_scan: bad argument");
  MsaHost H;
  int rc = msa_parse_checked("hhg_a3m_scan", rec, len, nullptr, mp, &H);
  if (rc != HHG_OK) return rc;
  *L = H.L; *N_in = H.N_in;
  if (has_ss) *has_ss = H.kss_pred >= 0;
  return HHG_OK;
}

static int msa_parse_impl(const char* rec, int64_t len, const hhg_seqdb* sq, const hhg_msa_params* mp, int32_t L_cap,
                          int32_t N_cap, int32_t* dims, uint8_t* X, uint16_t* I, int8_t* keep, int32_t* nres, int32_t* ksort) {
  if (!rec || len <= 0 || !dims || !X) return fail(HHG_EINVAL, "hhg_a3m_parse: bad argument");
  MsaHost H;
  int rc = msa_parse_checked("hhg_a3m_parse", rec, len, sq, mp, &H);
  if (rc != HHG_OK) return rc;
  msa_dims(H, dims);
  if (H.L > L_cap || H.N_in > N_cap) return fail(HHG_EINVAL, "hhg_a3m_parse: %d columns / %d sequences exceed the caller's capacity", H.L, H.N_in);
  const int L = H.L, N = H.N_in;
  for (int k = 0; k < N; ++k) {
    for (int i = 0; i <= L + 1; ++i) X[(size_t)k * (L + 2) + i] = H.X[(size_t)k * H.stride + i] & 0x7f;
    if (I) for (int i = 0; i <= L + 1; ++i) I[(size_t)k * (L + 2) + i] = 0;
    if (keep) keep[k] = H.keep[k];
    if (nres) nres[k] = H.nres[k];
    if (ksort) ksort[k] = H.ksort[k];
  }
  if (I)
    for (int i = 0; i <= L; ++i)
      for (uint32_t e = H.ins_off[i]; e < H.ins_off[i + 1]; ++e) I[(size_t)H.ins_k[e] * (L + 2) + i] = H.ins_cnt[e];
  return HHG_OK;
}

int hhg_a3m_parse(const char* rec, int64_t len, const hhg_msa_params* mp, int32_t L_cap, int32_t N_cap, int32_t* dims,
                  uint8_t* X, uint16_t* I, int8_t* keep, int32_t* nres, int32_t* ksort) {
  return msa_parse_impl(rec, len, nullptr, mp, L_cap, N_cap, dims, X, I, keep, nres, ksort);
}

int hhg_ca3m_parse(const char* rec, int64_t len, const hhg_seqdb* seqs, const hhg_msa_params* mp, int32_t L_cap, int32_t N_cap,
                   int32_t* dims, uint8_t* X, uint16_t* I, int8_t* keep, int32_t* nres, int32_t* ksort) {
  if (!seqs) return fail(HHG_EINVAL, "hhg_ca3m_parse: the sequence database is NULL");
  return msa_parse_impl(rec, len, seqs, mp, L_cap, N_cap, dims, X, I, keep, nres, ksort);
}

static int msa_to_hmm_impl(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_seqdb* sq, const hhg_msa_params* mp,
                           const float* S, const float* pb, int32_t L_cap, int32_t N_cap, int32_t* dims, int8_t* keep,
                           float* wg, float* f, float* tr, float* neff, float* neff_hmm, uint8_t* ss) {
  if (!ctx || !rec || len <= 0 || !pb || !dims || !f || !tr || !neff || !neff_hmm)
    return fail(HHG_EINVAL, "hhg_msa_to_hmm: bad argument");
  if (!ctx->msa_cache) ctx->msa_cache = std::make_shared<MsaChunk>();      // device buffers persist between calls
  MsaChunk& C = *std::static_pointer_cast<MsaChunk>(ctx->msa_cache);
  C.host.clear();
  C.host.resize(1);
  int rc = msa_parse_checked("hhg_msa_to_hmm", rec, len, sq, mp, &C.host[0]);
  if (rc != HHG_OK) return rc;
  if (mp->qsc > -10.f && !S) return fail(HHG_EINVAL, "hhg_msa_to_hmm: the qsc filter needs the substitution matrix S");
  CK(cudaSetDevice(ctx->device));
  const MsaHost& H = C.host[0];
  msa_dims(H, dims);
  if (H.L > L_cap || H.N_in > N_cap) return fail(HHG_EINVAL, "hhg_msa_to_hmm: %d columns / %d sequences exceed the caller's capacity %d / %d", H.L, H.N_in, L_cap, N_cap);
  rc = msa_chunk_run(ctx, C, *mp, S, pb, nullptr);
  if (rc != HHG_OK) return rc;
  const int L = H.L, N = H.N_in;
  int nf = 0;
  CK(cudaMemcpyAsync(&nf, C.nfil.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
  if (keep) CK(cudaMemcpyAsync(keep, C.keep.p, (size_t)N, cudaMemcpyDeviceToHost, ctx->stream));
  if (wg) CK(cudaMemcpyAsync(wg, C.wg.p, (size_t)N * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(f, C.f.p, (size_t)(L + 2) * 80, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(tr, C.tr.p, (size_t)(L + 1) * 28, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(neff, C.nm.p, (size_t)(L + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(neff + (L + 1), C.ni_f.p, (size_t)(L + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(neff + 2 * (L + 1), C.nd.p, (size_t)(L + 1) * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(neff_hmm, C.nhmm.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  dims[2] = nf;
  if (ss) { ss[0] = 0; msa_ss_bytes(H, ss + 1); ss[L + 1] = 0; }
  return HHG_OK;
}

int hhg_msa_to_hmm(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_msa_params* mp, const float* S, const float* pb,
                   int32_t L_cap, int32_t N_cap, int32_t* dims, int8_t* keep, float* wg, float* f, float* tr,
                   float* neff, float* neff_hmm, uint8_t* ss) {
  return msa_to_hmm_impl(ctx, rec, len, nullptr, mp, S, pb, L_cap, N_cap, dims, keep, wg, f, tr, neff, neff_hmm, ss);
}

int hhg_ca3m_to_hmm(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_seqdb* seqs, const hhg_msa_params* mp,
                    const float* S, const float* pb, int32_t L_cap, int32_t N_cap, int32_t* dims, int8_t* keep, float* wg,
                    float* f, float* tr, float* neff, float* neff_hmm) {
  if (!seqs) return fail(HHG_EINVAL, "hhg_ca3m_to_hmm: the sequence database is NULL");
  return msa_to_hmm_impl(ctx, rec, len, seqs, mp, S, pb, L_cap, N_cap, dims, keep, wg, f, tr, neff, neff_hmm, nullptr);
}

int hhg_ca3m_scan(const char* rec, int64_t len, const hhg_seqdb* seqs, const hhg_msa_params* mp, int32_t* L, int32_t* N_in) {
  if (!rec || len <= 0 || !L || !N_in || !seqs) return fail(HHG_EINVAL, "hhg_ca3m_scan: bad argument");
  MsaHost H;
  int rc = msa_parse_checked("hhg_ca3m_scan", rec, len, seqs, mp, &H);
  if (rc != HHG_OK) return rc;
  *L = H.L; *N_in = H.N_in;
  return HHG_OK;
}

// The records of an ffindex: record r is the len[r] bytes at data + off[r].
struct RecText {
  const char* data;
  const int64_t* off;
  const int64_t* len;
};

// Alignment records -> raw column records and pav, one group at a time: scan() parses a group on the host threads,
// build() runs filter / weights / M state / finish, k_msa_prepare and k_hhm_pav and writes the group's records to dst
// (in group order, each record's columns contiguous) and its pav rows to pav.  The A3M / CA3M shard loader and the
// stage of a record-sourced shard (hhg_db_stage) both go through it; host memory holds one group of parsed alignments.
struct MsaBuilder {
  hhg_ctx* ctx = nullptr;
  RecText T{};
  const hhg_seqdb* sq = nullptr;       // non-NULL: compressed A3M
  const hhg_msa_params* mp = nullptr;
  const float* S = nullptr;
  const float* pb = nullptr;
  const hhg_prep_params* pp = nullptr;
  HhmPrepArgs A{};
  MsaChunk C;
  DevBuf<long long> d_rec_off;
  DevBuf<uint8_t> d_ss;
  DevBuf<float> d_tau;
  DevBuf<int> d_L;
  std::vector<int32_t> rec, L;         // the scanned group: record indices and their lengths
  std::vector<long long> rec_off;      // first output column of each record of the group
  long long cols = 0;
  bool any_ss = false;                 // some record scanned so far predicts secondary structure

  // end of the group that starts at r[k0] of r[0..n): 256 MB of input text or max_records records
  int group_end(const int32_t* r, int k0, int n, const int32_t*) const {
    const long long kGroupText = 256ll << 20;
    int max_records = 8192;
    { const char* e = getenv("HHG_MSA_CHUNK_RECORDS"); if (e && atoi(e) > 0) max_records = atoi(e); }   // test knob: many small groups
    int k1 = k0;
    long long bytes = 0;
    while (k1 < n && k1 - k0 < max_records && (bytes == 0 || bytes + T.len[r[k1]] <= kGroupText)) bytes += T.len[r[k1++]];
    return k1;
  }
  // the lengths come from the full parse of scan()
  int peek(const int32_t*, int, int32_t*) { return HHG_OK; }

  int scan(const int32_t* r, int m) {
    rec.clear();
    C.host.clear();
    C.host.resize(m);
    const HostFail bad = host_for(m, [&](int k) -> std::string {
      if (T.len[r[k]] <= 0) return "empty record";
      return msa_parse_any(T.data + T.off[r[k]], T.len[r[k]], sq, mp, &C.host[k]);
    });
    if (bad.k >= 0) return fail(HHG_EINVAL, "record %d: %s", r[bad.k], bad.msg.c_str());
    L.resize(m);
    rec_off.resize(m);
    cols = 0;
    for (int k = 0; k < m; ++k) {
      const int Lk = C.host[k].L;
      if (Lk < 1 || Lk > 32767) return fail(HHG_EINVAL, "record %d: length %d out of [1,32767]", r[k], Lk);
      L[k] = Lk;
      rec_off[k] = cols; cols += Lk;
      any_ss |= C.host[k].kss_pred >= 0;
    }
    rec.assign(r, r + m);
    return HHG_OK;
  }

  // ss: write the ss bytes of the records (else 0); d_tr_full: hhg_query_from_a3m's linear transitions (one record);
  // neff_out: Neff_HMM of each record (host)
  int build(bool ss, ColRec* dst, float* pav, float* d_tr_full, float* neff_out) {
    const int m = (int)rec.size();
    const bool tau_on_host = pp->pcm == 2 && pp->pcc != 1.0f;
    int rc = msa_chunk_run(ctx, C, *mp, S, pb, rec.data());
    if (rc != HHG_OK) return rc;
    std::vector<uint8_t> ssb((size_t)cols, 0);
    if (ss) for (int k = 0; k < m; ++k) msa_ss_bytes(C.host[k], ssb.data() + rec_off[k]);
    CK(d_rec_off.ensure(m)); CK(d_ss.ensure((size_t)cols)); CK(d_L.ensure(m));
    CK(cudaMemcpyAsync(d_rec_off.p, rec_off.data(), (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_ss.p, ssb.data(), (size_t)cols, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_L.p, L.data(), (size_t)m * 4, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<float> tau_h;
    if (tau_on_host) {
      std::vector<float> nm((size_t)C.col_total);
      CK(cudaMemcpyAsync(nm.data(), C.nm.p, nm.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
      tau_h.resize((size_t)cols);
      for (int k = 0; k < m; ++k)
        for (int j = 1; j <= C.host[k].L; ++j)
          tau_h[(size_t)rec_off[k] + j - 1] = column_tau(pp, nm[(size_t)C.desc[k].col_off + j]);
      CK(d_tau.ensure((size_t)cols));
      CK(cudaMemcpyAsync(d_tau.p, tau_h.data(), (size_t)cols * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    const int threads = 128;
    k_msa_prepare<<<(unsigned)((cols + threads - 1) / threads), threads, 0, ctx->stream>>>(
        m, C.d_desc.p, d_rec_off.p, C.A, d_ss.p, A, ctx->lg2.p, ctx->diff.p, dst, cols, d_tr_full,
        tau_on_host ? d_tau.p : nullptr);
    k_hhm_pav<<<(unsigned)(((long long)m * 32 + threads - 1) / threads), threads, 0, ctx->stream>>>(
        m, d_L.p, d_rec_off.p, dst, nullptr, C.nhmm.p, A, pav, C.pb.p);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (neff_out) CK(cudaMemcpyAsync(neff_out, C.nhmm.p, (size_t)m * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));     // host staging of the group is reused by the next one
    return HHG_OK;
  }
};

// The parameter checks of the alignment loaders; `who` prefixes an error.
static int msa_load_args(const char* who, const hhg_seqdb* sq, const hhg_msa_params* mp, const float* S,
                         const hhg_prep_params* pp, const float* R, HhmPrepArgs* A) {
  int rc = msa_params_check(mp);
  if (rc != HHG_OK) return rc;
  if ((rc = seqdb_check(sq)) != HHG_OK) return rc;
  if (mp->qsc > -10.f && !S) return fail(HHG_EINVAL, "%s: the qsc filter needs the substitution matrix S", who);
  return hhm_prep_args(who, pp, R, A);
}

static int db_create_a3m_impl(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                              const hhg_seqdb* sq, const hhg_msa_params* mp, const float* S, const float* pb,
                              const hhg_prep_params* pp, const float* R, hhg_db** out, float* d_tr_full,
                              float* neff_hmm_out) {
  if (!ctx || !out || n <= 0 || !data || !off || !len || !pp || !R || !pb)
    return fail(HHG_EINVAL, "hhg_db_create_a3m: bad argument");
  MsaBuilder B;
  int rc = msa_load_args("hhg_db_create_a3m", sq, mp, S, pp, R, &B.A);
  if (rc != HHG_OK) return rc;
  B.ctx = ctx; B.T = RecText{data, off, len}; B.sq = sq; B.mp = mp; B.S = S; B.pb = pb; B.pp = pp;
  CK(cudaSetDevice(ctx->device));
  const bool timing = getenv("HHG_TIMING") != nullptr;
  const auto t_begin = std::chrono::steady_clock::now();
  double ms_scan = 0.0, ms_kernels = 0.0;

  // The records go through in groups of the builder; each group's column records land in a device piece and the
  // shard is assembled from the pieces at the end (a database of alignments is far larger than the shard it turns into).
  struct Piece { DevBuf<float4> cols; DevBuf<float> pav; int first = 0, n = 0; long long ncols = 0; };
  std::vector<std::unique_ptr<Piece>> pieces;
  std::vector<int32_t> Ls(n), all(n);
  std::iota(all.begin(), all.end(), 0);
  int t0 = 0;
  while (t0 < n) {
    const int t1 = B.group_end(all.data(), t0, n, nullptr);
    const int m = t1 - t0;
    const auto t_s0 = std::chrono::steady_clock::now();
    if ((rc = B.scan(all.data() + t0, m)) != HHG_OK) return rc;
    std::copy(B.L.begin(), B.L.end(), Ls.begin() + t0);
    ms_scan += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_s0).count();
    const auto t_c0 = std::chrono::steady_clock::now();
    pieces.emplace_back(new Piece());
    Piece& P = *pieces.back();
    P.first = t0; P.n = m; P.ncols = B.cols;
    CK(P.cols.alloc((size_t)B.cols * 7));
    CK(P.pav.alloc((size_t)m * 20));
    rc = B.build(true, reinterpret_cast<ColRec*>(P.cols.p), P.pav.p, d_tr_full, neff_hmm_out ? neff_hmm_out + t0 : nullptr);
    if (rc != HHG_OK) return rc;
    ms_kernels += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_c0).count();
    t0 = t1;
  }
  std::unique_ptr<hhg_db> holder;
  rc = db_new(ctx, n, Ls.data(), true, "record", &holder);
  if (rc != HHG_OK) return rc;
  hhg_db* db = holder.get();
  db->has_ss = B.any_ss;
  long long at = 0;
  for (auto& pc : pieces) {
    CK(cudaMemcpyAsync(db->cols_raw.p + (size_t)at * 7, pc->cols.p, (size_t)pc->ncols * 7 * sizeof(float4), cudaMemcpyDeviceToDevice, ctx->stream));
    CK(cudaMemcpyAsync(db->pav.p + (size_t)pc->first * 20, pc->pav.p, (size_t)pc->n * 80, cudaMemcpyDeviceToDevice, ctx->stream));
    at += pc->ncols;
  }
  rc = db_publish_raw(ctx, holder, out);
  if (rc != HHG_OK) return rc;
  pieces.clear();
  if (timing) {
    const double ms_all = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
    fprintf(stderr, "[hhg] alignment loader: %d records, host scan %.1f ms, kernels %.1f ms, rest (copies) %.1f ms\n",
            n, ms_scan, ms_kernels, ms_all - ms_scan - ms_kernels);
  }
  return HHG_OK;
}

int hhg_db_create_a3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                      const hhg_msa_params* mp, const float* S, const float* pb, const hhg_prep_params* pp,
                      const float* R, hhg_db** out) {
  return db_create_a3m_impl(ctx, n, data, off, len, nullptr, mp, S, pb, pp, R, out, nullptr, nullptr);
}

int hhg_db_create_ca3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len, const hhg_seqdb* seqs,
                       const hhg_msa_params* mp, const float* S, const float* pb, const hhg_prep_params* pp,
                       const float* R, hhg_db** out) {
  if (!seqs) return fail(HHG_EINVAL, "hhg_db_create_ca3m: the sequence database is NULL");
  return db_create_a3m_impl(ctx, n, data, off, len, seqs, mp, S, pb, pp, R, out, nullptr, nullptr);
}

int hhg_hhm_scan(const char* rec, int64_t len, int32_t* L, int32_t* has_ss) {
  if (!rec || len <= 0 || !L || !has_ss) return fail(HHG_EINVAL, "hhg_hhm_scan: bad argument");
  HhmScanner sc(rec, len);
  if (!sc.peek(L, has_ss)) return fail(HHG_EINVAL, "hhg_hhm_scan: no LENG line / not an HHM record");
  return HHG_OK;
}

int hhg_hhm_parse(const char* rec, int64_t len, int32_t L, int32_t* f_mb, int32_t* trn_mb, uint8_t* ss,
                  int32_t* null_mb, float* neff_hmm, int32_t* has_pc) {
  if (!rec || len <= 0 || L < 1 || !f_mb || !trn_mb || !ss || !null_mb || !neff_hmm || !has_pc)
    return fail(HHG_EINVAL, "hhg_hhm_parse: bad argument");
  HhmScanner sc(rec, len);
  std::string msg = sc.parse(L, f_mb, trn_mb, ss, null_mb, neff_hmm, has_pc);
  if (!msg.empty()) return fail(HHG_EINVAL, "hhg_hhm_parse: %s", msg.c_str());
  return HHG_OK;
}

// HHM records -> raw column records and pav, one chunk at a time (the shape of MsaBuilder): peek() reads the LENG
// lines, scan() parses a chunk on the host threads, build() runs k_hhm_prepare and k_hhm_pav and writes the chunk's
// records to dst and its pav rows to pav.  The HHM shard loader and the stage of a record-sourced shard both use it.
struct HhmBuilder {
  hhg_ctx* ctx = nullptr;
  RecText T{};
  const hhg_prep_params* pp = nullptr;
  HhmPrepArgs A{};
  HhmStaging st;
  DevBuf<int32_t> d_f, d_trn, d_null, d_haspc, d_L;
  DevBuf<uint8_t> d_ss;
  DevBuf<float> d_neff, d_tau;
  DevBuf<long long> d_coff;
  std::vector<int32_t> rec, L;         // the scanned chunk: record indices and their lengths
  std::vector<long long> rec_off;      // first output column of each record of the chunk
  long long cols = 0;
  bool any_ss = false;                 // some record peeked so far predicts secondary structure

  // end of the chunk that starts at r[k0] of r[0..n): 2 M columns; Lrec: lengths by record index
  int group_end(const int32_t* r, int k0, int n, const int32_t* Lrec) const {
    const long long kChunkCols = 2000000;
    int k1 = k0;
    long long c = 0;
    while (k1 < n && (c == 0 || c + Lrec[r[k1]] <= kChunkCols)) c += Lrec[r[k1++]];
    return k1;
  }
  // LENG of records r[0..m) into Lout[0..m) (not range checked) and whether any predicts secondary structure
  int peek(const int32_t* r, int m, int32_t* Lout) {
    for (int k = 0; k < m; ++k) {
      int32_t has_ss = 0;
      HhmScanner sc(T.data + T.off[r[k]], T.len[r[k]]);
      if (T.len[r[k]] <= 0 || !sc.peek(&Lout[k], &has_ss)) return fail(HHG_EINVAL, "record %d: no LENG line / not an HHM record", r[k]);
      any_ss |= has_ss != 0;
    }
    return HHG_OK;
  }

  int scan(const int32_t* r, int m) {
    rec.clear();
    L.resize(m);
    int rc = peek(r, m, L.data());
    if (rc != HHG_OK) return rc;
    rec_off.resize(m);
    cols = 0;
    for (int k = 0; k < m; ++k) { rec_off[k] = cols; cols += L[k]; }
    st.f_mb.assign((size_t)cols * 20, 0);
    st.trn_mb.assign((size_t)(cols + m) * 10, 0);
    st.ss.assign((size_t)cols, 0);
    st.null_mb.assign((size_t)m * 20, 0);
    st.neff_hmm.assign(m, 0.f);
    st.has_pc.assign(m, 0);
    const HostFail bad = host_for(m, [&](int k) {
      HhmScanner sc(T.data + T.off[r[k]], T.len[r[k]]);
      return sc.parse(L[k], st.f_mb.data() + (size_t)rec_off[k] * 20,
                      st.trn_mb.data() + (size_t)(rec_off[k] + k) * 10, st.ss.data() + rec_off[k],
                      st.null_mb.data() + (size_t)k * 20, &st.neff_hmm[k], &st.has_pc[k]);
    });
    if (bad.k >= 0) return fail(HHG_EINVAL, "record %d: %s", r[bad.k], bad.msg.c_str());
    rec.assign(r, r + m);
    return HHG_OK;
  }

  // ss: write the ss bytes of the records (else 0); d_tr_full: hhg_query_from_hhm's linear transitions (one record);
  // neff_out: Neff_HMM of each record (host)
  int build(bool ss, ColRec* dst, float* pav, float* d_tr_full, float* neff_out) {
    const int m = (int)rec.size();
    const bool tau_on_host = pp->pcm == 2 && pp->pcc != 1.0f;   // needs the C library's powf: computed per column here
    CK(d_f.ensure(st.f_mb.size())); CK(d_trn.ensure(st.trn_mb.size())); CK(d_ss.ensure(st.ss.size()));
    CK(d_null.ensure(st.null_mb.size())); CK(d_haspc.ensure(m)); CK(d_neff.ensure(m)); CK(d_coff.ensure(m)); CK(d_L.ensure(m));
    CK(cudaMemcpyAsync(d_f.p, st.f_mb.data(), st.f_mb.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_trn.p, st.trn_mb.data(), st.trn_mb.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_ss.p, st.ss.data(), st.ss.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_null.p, st.null_mb.data(), st.null_mb.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_haspc.p, st.has_pc.data(), (size_t)m * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_neff.p, st.neff_hmm.data(), (size_t)m * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_coff.p, rec_off.data(), (size_t)m * 8, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(d_L.p, L.data(), (size_t)m * 4, cudaMemcpyHostToDevice, ctx->stream));
    std::vector<float> tau_h;
    if (tau_on_host) {
      tau_h.resize((size_t)cols);
      for (int k = 0; k < m; ++k) {
        const int32_t* rows = st.trn_mb.data() + (size_t)(rec_off[k] + k) * 10;
        for (int j = 1; j <= L[k]; ++j) {
          const float nM = (float)rows[(size_t)j * 10 + 7] / 1000.0f;
          tau_h[(size_t)rec_off[k] + j - 1] = column_tau(pp, nM);
        }
      }
      CK(d_tau.ensure((size_t)cols));
      CK(cudaMemcpyAsync(d_tau.p, tau_h.data(), (size_t)cols * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    const int threads = 128;
    k_hhm_prepare<<<(unsigned)((cols + threads - 1) / threads), threads, 0, ctx->stream>>>(
        m, d_L.p, d_coff.p, d_f.p, d_trn.p, ss ? d_ss.p : nullptr, d_haspc.p, A, ctx->lg2.p,
        ctx->diff.p, dst, cols, d_tr_full, tau_on_host ? d_tau.p : nullptr);
    k_hhm_pav<<<(unsigned)(((long long)m * 32 + threads - 1) / threads), threads, 0, ctx->stream>>>(
        m, d_L.p, d_coff.p, dst, d_null.p, d_neff.p, A, pav);
    ctx->launches += 2;
    CK(cudaGetLastError());
    if (neff_out) memcpy(neff_out, st.neff_hmm.data(), (size_t)m * 4);
    CK(cudaStreamSynchronize(ctx->stream));   // staging is reused by the next chunk
    return HHG_OK;
  }
};

static int db_create_hhm_impl(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                              const hhg_prep_params* pp, const float* R, hhg_db** out, float* d_tr_full) {
  if (!ctx || !out || n <= 0 || !data || !off || !len || !pp || !R)
    return fail(HHG_EINVAL, "hhg_db_create_hhm: bad argument");
  HhmBuilder B;
  int rc = hhm_prep_args("hhg_db_create_hhm", pp, R, &B.A);
  if (rc != HHG_OK) return rc;
  B.ctx = ctx; B.T = RecText{data, off, len}; B.pp = pp;
  CK(cudaSetDevice(ctx->device));
  // pass 1: lengths (LENG) and whether any record predicts secondary structure
  std::vector<int32_t> Ls(n), all(n);
  std::iota(all.begin(), all.end(), 0);
  if ((rc = B.peek(all.data(), n, Ls.data())) != HHG_OK) return rc;
  const bool any_ss = B.any_ss;
  std::unique_ptr<hhg_db> holder;
  if ((rc = db_new(ctx, n, Ls.data(), true, "record", &holder)) != HHG_OK) return rc;
  hhg_db* db = holder.get();
  db->has_ss = any_ss;
  // pass 2: chunks of records -> host staging (parsed by a few threads) -> device -> k_hhm_prepare / k_hhm_pav
  int t0 = 0;
  while (t0 < n) {
    const int t1 = B.group_end(all.data(), t0, n, Ls.data());
    if ((rc = B.scan(all.data() + t0, t1 - t0)) != HHG_OK) return rc;
    // d_tr_full only with a single chunk (hhg_query_from_hhm: one record)
    rc = B.build(any_ss, reinterpret_cast<ColRec*>(db->cols_raw.p) + db->col_off[t0], db->pav.p + (size_t)t0 * 20, d_tr_full, nullptr);
    if (rc != HHG_OK) return rc;
    t0 = t1;
  }
  return db_publish_raw(ctx, holder, out);
}

int hhg_db_create_hhm(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                      const hhg_prep_params* pp, const float* R, hhg_db** out) {
  return db_create_hhm_impl(ctx, n, data, off, len, pp, R, out, nullptr);
}

// PrepareQueryHMM for an HHM query without context-specific pseudocounts (par.nocontxt; src/hhfunc.cpp:121-160): the
// same three steps a template gets -- AddTransitionPseudocounts, PreparePseudocounts + AddAminoAcidPseudocounts,
// CalculateAminoAcidBackground -- so the record runs through the database loader's kernels and comes back as the host
// arrays hhg_query_set / hhg_prefilter_build_profile take.
int hhg_query_from_hhm(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_prep_params* pp, const float* R,
                       int32_t L_cap, int32_t* L_out, float* p, float* tr, uint8_t* ss, float* pav, float* neff) {
  if (!ctx || !rec || len <= 0 || !pp || !R || !L_out || !p || !tr || !pav) return fail(HHG_EINVAL, "hhg_query_from_hhm: bad argument");
  int32_t L = 0, has_ss = 0;
  { HhmScanner sc(rec, len); if (!sc.peek(&L, &has_ss)) return fail(HHG_EINVAL, "hhg_query_from_hhm: not an HHM record"); }
  if (L < 1 || L > L_cap) return fail(HHG_EINVAL, "hhg_query_from_hhm: query length %d exceeds the caller's capacity %d", L, L_cap);
  CK(cudaSetDevice(ctx->device));
  DevBuf<float> d_tr;
  CK(d_tr.alloc((size_t)(L + 1) * 7));
  hhg_db* db = nullptr;
  const int64_t zero = 0;
  int rc = db_create_hhm_impl(ctx, 1, rec, &zero, &len, pp, R, &db, d_tr.p);
  if (rc != HHG_OK) return rc;
  std::unique_ptr<hhg_db> holder(db);
  if ((rc = query_from_shard(ctx, db, L, d_tr.p, p, tr, ss, pav)) != HHG_OK) return rc;
  if (neff) {
    std::vector<int32_t> f((size_t)L * 20), trn((size_t)(L + 1) * 10), nul(20);
    std::vector<uint8_t> ssb(L);
    int32_t has_pc = 0;
    rc = hhg_hhm_parse(rec, len, L, f.data(), trn.data(), ssb.data(), nul.data(), neff, &has_pc);
    if (rc != HHG_OK) return rc;
  }
  *L_out = L;
  return HHG_OK;
}

// The same for a query ALIGNMENT (hhblits: ReadQueryFile -> Alignment::Read / Compress / Filter /
// FrequenciesAndTransitions, src/hhblits.cpp:1424-1453, then PrepareQueryHMM's nocontxt branch).
int hhg_query_from_a3m(hhg_ctx* ctx, const char* rec, int64_t len, const hhg_msa_params* mp, const float* S, const float* pb,
                       const hhg_prep_params* pp, const float* R, int32_t L_cap, int32_t* L_out, float* p, float* tr,
                       uint8_t* ss, float* pav, float* neff) {
  if (!ctx || !rec || len <= 0 || !pp || !R || !pb || !L_out || !p || !tr || !pav) return fail(HHG_EINVAL, "hhg_query_from_a3m: bad argument");
  int32_t L = 0, N = 0, has_ss = 0;
  int rc = hhg_a3m_scan(rec, len, mp, &L, &N, &has_ss);
  if (rc != HHG_OK) return rc;
  if (L < 1 || L > L_cap) return fail(HHG_EINVAL, "hhg_query_from_a3m: query length %d exceeds the caller's capacity %d", L, L_cap);
  CK(cudaSetDevice(ctx->device));
  DevBuf<float> d_tr;
  CK(d_tr.alloc((size_t)(L + 1) * 7));
  hhg_db* db = nullptr;
  const int64_t zero = 0;
  float nh = 0.f;
  rc = db_create_a3m_impl(ctx, 1, rec, &zero, &len, nullptr, mp, S, pb, pp, R, &db, d_tr.p, &nh);
  if (rc != HHG_OK) return rc;
  std::unique_ptr<hhg_db> holder(db);
  if ((rc = query_from_shard(ctx, db, L, d_tr.p, p, tr, ss, pav)) != HHG_OK) return rc;
  if (neff) *neff = nh;
  *L_out = L;
  return HHG_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Context-specific pseudocounts of the query (hhg_crf.cuh)
// One handle for either engine, as the reference holds one Pseudocounts* whatever the file type: host.library tells
// which score kernel runs (k_crf_scores or k_lib_scores) and where the tail's maximum starts.
struct hhg_crf {
  int device = 0;
  hhg::CrfHost host;
  DevBuf<double> d_w, d_bias, d_ww;
};

static int crf_upload(hhg_ctx* ctx, std::unique_ptr<hhg_crf>& c, hhg_crf** out) {
  CK(cudaSetDevice(ctx->device));
  c->device = ctx->device;
  CK(c->d_w.alloc(c->host.w.size())); CK(c->d_bias.alloc(c->host.bias.size()));
  CK(cudaMemcpyAsync(c->d_w.p, c->host.w.data(), c->host.w.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(c->d_bias.p, c->host.bias.data(), c->host.bias.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  if (c->host.library) {
    CK(c->d_ww.alloc(c->host.ww.size()));
    CK(cudaMemcpyAsync(c->d_ww.p, c->host.ww.data(), c->host.ww.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  *out = c.release();
  return HHG_OK;
}

int hhg_crf_create(hhg_ctx* ctx, const char* text, int64_t len, hhg_crf** out) {
  if (!ctx || !text || len <= 0 || !out) return fail(HHG_EINVAL, "hhg_crf_create: bad argument");
  std::unique_ptr<hhg_crf> c(new hhg_crf());
  const std::string msg = crf_parse(text, len, &c->host);
  if (!msg.empty()) return fail(HHG_EINVAL, "hhg_crf_create: %s", msg.c_str());
  return crf_upload(ctx, c, out);
}

int hhg_context_library_create(hhg_ctx* ctx, const char* text, int64_t len, double weight_center, double weight_decay,
                               hhg_crf** out) {
  if (!ctx || !text || len <= 0 || !out) return fail(HHG_EINVAL, "hhg_context_library_create: bad argument");
  std::unique_ptr<hhg_crf> c(new hhg_crf());
  const std::string msg = lib_parse(text, len, weight_center, weight_decay, &c->host);
  if (!msg.empty()) return fail(HHG_EINVAL, "hhg_context_library_create: %s", msg.c_str());
  return crf_upload(ctx, c, out);
}

int hhg_crf_destroy(hhg_crf* crf) { delete crf; return HHG_OK; }

int hhg_crf_info(const hhg_crf* crf, int32_t* n_states, int32_t* window, double* pc /* [n_states*20] or NULL */) {
  if (!crf || !n_states || !window) return fail(HHG_EINVAL, "hhg_crf_info: bad argument");
  *n_states = crf->host.K; *window = crf->host.W;
  if (pc) memcpy(pc, crf->host.pc.data(), crf->host.pc.size() * 8);
  return HHG_OK;
}

static double crf_tail_start(const hhg::CrfHost& h) { return h.library ? -FLT_MAX : -DBL_MAX; }

// Host only: the per-column tail of hhg_query_context_pseudocounts on caller-supplied context scores
// (score[L*K], what k_crf_scores produces), for inspection and CPU-side tests.
int hhg_crf_tail_host(const hhg_crf* crf, int32_t L, double* score, const float* f, const float* neff_m, const hhg_admix* admix,
                      float* p) {
  if (!crf || L < 1 || !score || !f || !neff_m || !admix || !p) return fail(HHG_EINVAL, "hhg_crf_tail_host: bad argument");
  const int K = crf->host.K;
  for (int i = 0; i < L; ++i) {
    double cnt[20];
    for (int a = 0; a < 20; ++a) cnt[a] = f[(size_t)(i + 1) * 20 + a] * neff_m[i + 1];
    crf_column_tail(K, crf_tail_start(crf->host), score + (size_t)i * K, crf->host.pc.data(), cnt, (double)neff_m[i + 1],
                    admix->kind, admix->pca, admix->pcb, admix->pcc, p + (size_t)(i + 1) * 20);
  }
  return HHG_OK;
}

// Host only: parse without a device (no upload); for CPU-side tests of the parser and the tail.
int hhg_crf_parse_host(const char* text, int64_t len, hhg_crf** out) {
  if (!text || len <= 0 || !out) return fail(HHG_EINVAL, "hhg_crf_parse_host: bad argument");
  std::unique_ptr<hhg_crf> c(new hhg_crf());
  const std::string msg = crf_parse(text, len, &c->host);
  if (!msg.empty()) return fail(HHG_EINVAL, "hhg_crf_parse_host: %s", msg.c_str());
  *out = c.release();
  return HHG_OK;
}

int hhg_context_library_parse_host(const char* text, int64_t len, double weight_center, double weight_decay, hhg_crf** out) {
  if (!text || len <= 0 || !out) return fail(HHG_EINVAL, "hhg_context_library_parse_host: bad argument");
  std::unique_ptr<hhg_crf> c(new hhg_crf());
  const std::string msg = lib_parse(text, len, weight_center, weight_decay, &c->host);
  if (!msg.empty()) return fail(HHG_EINVAL, "hhg_context_library_parse_host: %s", msg.c_str());
  *out = c.release();
  return HHG_OK;
}

// Host only: weights of one state, w[window*20] (row-major window x amino acid) and its bias.
int hhg_crf_state(const hhg_crf* crf, int32_t k, double* w, double* bias) {
  if (!crf || k < 0 || k >= crf->host.K || !w || !bias) return fail(HHG_EINVAL, "hhg_crf_state: bad argument");
  for (int j = 0; j < crf->host.W; ++j)
    for (int a = 0; a < 20; ++a) w[j * 20 + a] = crf->host.w[((size_t)j * 20 + a) * crf->host.K + k];
  *bias = crf->host.bias[k];
  return HHG_OK;
}

int hhg_query_context_pseudocounts(hhg_ctx* ctx, const hhg_crf* crf, int32_t L, const float* f, const float* neff_m,
                                   float neff_hmm, const float* pb, const hhg_admix* admix, float* p, float* pav) {
  if (!ctx || !crf || L < 1 || !f || !neff_m || !admix || !p) return fail(HHG_EINVAL, "hhg_query_context_pseudocounts: bad argument");
  if (admix->kind < 0 || admix->kind > 2) return fail(HHG_EINVAL, "hhg_query_context_pseudocounts: admixture kind %d (0 constant, 1 CS-BLAST, 2 HHsearch)", admix->kind);
  if (pav && !pb) return fail(HHG_EINVAL, "hhg_query_context_pseudocounts: pav needs the background pb");
  // the result only feeds hhg_query_set, which takes Lq <= 32767; k_crf_scores runs one block row per column
  if (L > 32767) return fail(HHG_EINVAL, "hhg_query_context_pseudocounts: L = %d exceeds the query limit of 32767 columns", L);
  if (crf->device != ctx->device)
    return fail(HHG_EINVAL, "hhg_query_context_pseudocounts: the %s was created on device %d, the context is on device %d",
                crf->host.library ? "context library" : "CRF",
                crf->device, ctx->device);
  CK(cudaSetDevice(ctx->device));
  const int K = crf->host.K, W = crf->host.W;
  // HMM::fillCountProfile (src/hhhmm.cpp:1843-1849): counts = f * Neff_M (float product), neff = Neff_M
  std::vector<double> counts((size_t)L * 20), neff(L);
  for (int i = 0; i < L; ++i) {
    neff[i] = neff_m[i + 1];
    for (int a = 0; a < 20; ++a) counts[(size_t)i * 20 + a] = f[(size_t)(i + 1) * 20 + a] * neff_m[i + 1];
  }
  struct CrfStage {
    DevBuf<double> counts, score;
    double* h_score = nullptr; size_t h_n = 0;
    ~CrfStage() { if (h_score) cudaFreeHost(h_score); }
  };
  if (!ctx->crf_cache) ctx->crf_cache = std::make_shared<CrfStage>();
  CrfStage& st = *std::static_pointer_cast<CrfStage>(ctx->crf_cache);
  const size_t ns = (size_t)L * K;
  CK(st.counts.ensure(counts.size())); CK(st.score.ensure(ns));
  if (st.h_n < ns) {
    if (st.h_score) cudaFreeHost(st.h_score);
    st.h_score = nullptr; st.h_n = 0;
    CK(cudaHostAlloc((void**)&st.h_score, ns * 8, cudaHostAllocDefault));
    st.h_n = ns;
  }
  CK(cudaMemcpyAsync(st.counts.p, counts.data(), counts.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  const dim3 grid((K + 255) / 256, L);
  if (crf->host.library)
    k_lib_scores<<<grid, 256, 0, ctx->stream>>>(L, K, W, crf->d_w.p, crf->d_bias.p, crf->d_ww.p, st.counts.p, st.score.p);
  else
    k_crf_scores<<<grid, 256, 0, ctx->stream>>>(L, K, W, crf->d_w.p, crf->d_bias.p, st.counts.p, st.score.p);
  ctx->launches++;
  CK(cudaGetLastError());
  double* score = st.h_score;
  CK(cudaMemcpyAsync(score, st.score.p, ns * 8, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  host_for(L, [&](int i) {
    crf_column_tail(K, crf_tail_start(crf->host), score + (size_t)i * K, crf->host.pc.data(), counts.data() + (size_t)i * 20, neff[i],
                    admix->kind, admix->pca, admix->pcb, admix->pcc, p + (size_t)(i + 1) * 20);
    return std::string();
  });
  if (pav) {                               // HMM::CalculateAminoAcidBackground (src/hhhmm.cpp:1854-1868)
    float pv[20];
    for (int a = 0; a < 20; ++a) pv[a] = pb[a] * 100.0f / neff_hmm;
    for (int i = 1; i <= L; ++i) for (int a = 0; a < 20; ++a) pv[a] += p[(size_t)i * 20 + a];
    float sum = 0.0f;
    for (int a = 0; a < 20; ++a) sum += pv[a];
    if (sum != 0.0f) { const float fac = 1.0 / sum; for (int a = 0; a < 20; ++a) pv[a] *= fac; }
    memcpy(pav, pv, 80);
    memcpy(p, pv, 80); memcpy(p + (size_t)(L + 1) * 20, pv, 80);
  }
  return HHG_OK;
}

// The resident binary format: column records before the null model + pav.  read_* copy it out (to be stored
// next to the ffindex files), hhg_db_create_packed loads it back without parsing anything.
int hhg_db_read_cols(hhg_ctx* ctx, const hhg_db* db, int which, int64_t first, int64_t count, void* out) {
  if (!ctx || !db || !out || first < 0 || count < 0 || first + count > db->total_cols)
    return fail(HHG_EINVAL, "hhg_db_read_cols: bad argument");
  if (which != 0 && which != 1) return fail(HHG_EINVAL, "hhg_db_read_cols: which must be 0 (raw) or 1 (prepared)");
  if (which == 0 && !db->raw) return fail(HHG_EINVAL, "hhg_db_read_cols: db holds no pre-null-model records");
  if (which == 1 && !db->prepared) return fail(HHG_EINVAL, "hhg_db_read_cols: call hhg_db_apply_null_model first");
  CK(cudaSetDevice(ctx->device));
  const ColRec* src = reinterpret_cast<const ColRec*>(which == 0 ? db->cols_raw.p : db->cols.p) + first;
  CK(cudaMemcpyAsync(out, src, (size_t)count * sizeof(ColRec), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

int hhg_db_read_pav(hhg_ctx* ctx, const hhg_db* db, float* out) {
  if (!ctx || !db || !out || !db->raw) return fail(HHG_EINVAL, "hhg_db_read_pav: bad argument / db not raw");
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(out, db->pav.p, (size_t)db->n * 20 * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

int hhg_db_create_packed(hhg_ctx* ctx, int n, const int32_t* L, const void* cols_raw, int has_ss,
                         const float* pav, hhg_db** out) {
  if (!ctx || !out || n <= 0 || !L || !cols_raw || !pav) return fail(HHG_EINVAL, "hhg_db_create_packed: bad argument");
  CK(cudaSetDevice(ctx->device));
  std::unique_ptr<hhg_db> holder;
  int rc = db_new(ctx, n, L, true, "target", &holder);
  if (rc != HHG_OK) return rc;
  hhg_db* db = holder.get();
  db->has_ss = has_ss != 0;
  CK(cudaMemcpyAsync(db->cols_raw.p, cols_raw, (size_t)db->total_cols * sizeof(ColRec), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(db->pav.p, pav, (size_t)n * 20 * 4, cudaMemcpyHostToDevice, ctx->stream));
  return db_publish_raw(ctx, holder, out);
}

int hhg_debug_fastlog2_table(hhg_ctx* ctx, float* lg2_out) {
  if (!ctx || !lg2_out) return fail(HHG_EINVAL, "bad argument");
  memcpy(lg2_out, ctx->h_lg2.data(), 1025 * 4);
  return HHG_OK;
}

int hhg_db_destroy(hhg_db* db) {
  if (db) {
    cudaSetDevice(db->device);
    if (db->store) db->store->users--;
    if (db->src) db->src->users--;
    delete db;
  }
  return HHG_OK;
}
int hhg_db_size(const hhg_db* db) { return db ? db->n : 0; }
long long hhg_db_columns(const hhg_db* db) { return db ? db->total_cols : 0; }

int hhg_db_lengths(const hhg_db* db, int32_t* out) {
  if (!db || !out) return fail(HHG_EINVAL, "hhg_db_lengths: bad argument");
  memcpy(out, db->L.data(), (size_t)db->n * sizeof(int32_t));
  return HHG_OK;
}


// ------------------------------------------------------------------------- host-resident store + staged shard
// HHEntry::getTemplateHMM reads only the prefilter's survivors (src/hhdatabase.cpp:300-336); here the records of all
// profiles sit in page-locked host memory and hhg_db_stage brings the survivors into a device cache (DESIGN 4.12).
int hhg_dbstore_create(hhg_ctx* ctx, int capacity_targets, long long capacity_cols, int has_ss, hhg_dbstore** out) {
  if (!ctx || !out || capacity_targets < 1 || capacity_cols < capacity_targets)
    return fail(HHG_EINVAL, "hhg_dbstore_create: bad argument (every target has at least one column)");
  CK(cudaSetDevice(ctx->device));
  std::unique_ptr<hhg_dbstore> st(new hhg_dbstore());
  st->device = ctx->device;
  st->has_ss = has_ss != 0;
  st->cap_targets = capacity_targets;
  st->cap_cols = capacity_cols;
  const unsigned flags = cudaHostAllocMapped | cudaHostAllocPortable;
  cudaError_t e1 = cudaHostAlloc((void**)&st->cols, (size_t)capacity_cols * sizeof(ColRec), flags);
  cudaError_t e2 = e1 == cudaSuccess ? cudaHostAlloc((void**)&st->pav, (size_t)capacity_targets * 80, flags) : e1;
  if (e2 != cudaSuccess) {
    if (e1 == cudaSuccess) cudaFreeHost(st->cols);
    cudaGetLastError();
    return fail(HHG_ENOMEM, "hhg_dbstore_create: cannot page-lock %.3f GB of host memory (%s)",
                ((double)capacity_cols * sizeof(ColRec) + (double)capacity_targets * 80) / 1e9, cudaGetErrorString(e2));
  }
  void *dc = nullptr, *dp = nullptr;
  cudaError_t e3 = cudaHostGetDevicePointer(&dc, st->cols, 0), e4 = cudaHostGetDevicePointer(&dp, st->pav, 0);
  if (e3 != cudaSuccess || e4 != cudaSuccess) {
    cudaFreeHost(st->cols); cudaFreeHost(st->pav);
    return fail(HHG_ECUDA, "hhg_dbstore_create: the device cannot map host memory");
  }
  st->d_cols = (const float4*)dc;
  st->d_pav = (const float*)dp;
  *out = st.release();
  return HHG_OK;
}

int hhg_dbstore_destroy(hhg_dbstore* store) {
  if (!store) return HHG_OK;
  if (store->users > 0) return fail(HHG_EINVAL, "hhg_dbstore_destroy: %d staged shards still use the store", store->users);
  cudaSetDevice(store->device);
  cudaFreeHost(store->cols);
  cudaFreeHost(store->pav);
  delete store;
  return HHG_OK;
}
int hhg_dbstore_size(const hhg_dbstore* store) { return store ? store->n : 0; }
long long hhg_dbstore_columns(const hhg_dbstore* store) { return store ? store->total_cols : 0; }
int hhg_dbstore_lengths(const hhg_dbstore* store, int32_t* out) {
  if (!store || !out) return fail(HHG_EINVAL, "hhg_dbstore_lengths: bad argument");
  memcpy(out, store->L.data(), (size_t)store->n * sizeof(int32_t));
  return HHG_OK;
}

// Checks that n more targets of lengths L fit and enters them in the store's tables; the caller then fills the records
// [first, first + sum(L)) and pav rows [n0, n0 + n).  Nothing changes when it fails.
static int dbstore_reserve(hhg_dbstore* st, const char* who, int n, const int32_t* L, long long* first) {
  long long cols = 0;
  for (int k = 0; k < n; ++k) {
    if (L[k] < 1 || L[k] > 32767) return fail(HHG_EINVAL, "%s: target %d: length %d out of [1,32767]", who, k, L[k]);
    cols += L[k];
  }
  if (st->n + (long long)n > st->cap_targets || st->total_cols + cols > st->cap_cols)
    return fail(HHG_EINVAL, "%s: %lld targets / %lld columns needed, the store was created for %d / %lld", who,
                st->n + (long long)n, st->total_cols + cols, st->cap_targets, st->cap_cols);
  *first = st->total_cols;
  for (int k = 0; k < n; ++k) {
    st->L.push_back(L[k]);
    st->col_off.push_back(st->total_cols);
    st->total_cols += L[k];
  }
  st->n += n;
  return HHG_OK;
}

int hhg_dbstore_append_packed(hhg_dbstore* store, int n, const int32_t* L, const void* cols_raw, const float* pav) {
  if (!store || n < 1 || !L || !cols_raw || !pav) return fail(HHG_EINVAL, "hhg_dbstore_append_packed: bad argument");
  const int n0 = store->n;
  long long first = 0;
  int rc = dbstore_reserve(store, "hhg_dbstore_append_packed", n, L, &first);
  if (rc != HHG_OK) return rc;
  memcpy(store->cols + first, cols_raw, (size_t)(store->total_cols - first) * sizeof(ColRec));
  memcpy(store->pav + (size_t)n0 * 20, pav, (size_t)n * 80);
  return HHG_OK;
}

int hhg_dbstore_append_db(hhg_ctx* ctx, hhg_dbstore* store, const hhg_db* db) {
  if (!ctx || !store || !db) return fail(HHG_EINVAL, "hhg_dbstore_append_db: bad argument");
  if (!db->raw || db->stage) return fail(HHG_EINVAL, "hhg_dbstore_append_db: the shard must be raw and not staged");
  if (db->has_ss != store->has_ss) return fail(HHG_EINVAL, "hhg_dbstore_append_db: shard and store differ in has_ss");
  if (db->device != ctx->device) return fail(HHG_EINVAL, "db lives on device %d, ctx on %d", db->device, ctx->device);
  const int n0 = store->n;
  long long first = 0;
  int rc = dbstore_reserve(store, "hhg_dbstore_append_db", db->n, db->L.data(), &first);
  if (rc != HHG_OK) return rc;
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(store->cols + first, db->cols_raw.p, (size_t)db->total_cols * sizeof(ColRec), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(store->pav + (size_t)n0 * 20, db->pav.p, (size_t)db->n * 80, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

// An empty staged shard of max_targets slots over an arena of max_cols records.
static int staged_new(hhg_ctx* ctx, int max_targets, long long max_cols, bool has_ss, std::unique_ptr<hhg_db>* out) {
  CK(cudaSetDevice(ctx->device));
  std::unique_ptr<hhg_db> db(new hhg_db());
  db->device = ctx->device;
  db->n = max_targets;
  db->total_cols = max_cols;
  db->has_ss = has_ss;
  db->L.assign(max_targets, 0);
  db->col_off.assign(max_targets, 0);
  db->raw = true;
  db->prepared = false;
  CK(db->cols.alloc((size_t)max_cols * 7));
  CK(db->cols_raw.alloc((size_t)max_cols * 7));
  CK(db->pav.alloc((size_t)max_targets * 20));
  CK(db->dL.alloc(max_targets));
  CK(db->dcol_off.alloc(max_targets));
  CK(db->d_slot_id.alloc(max_targets));
  CK(db->d_zero.alloc(max_targets));
  std::vector<int> ident(max_targets);
  std::iota(ident.begin(), ident.end(), 0);
  CK(cudaMemcpyAsync(db->d_slot_id.p, ident.data(), (size_t)max_targets * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(db->d_zero.p, 0, (size_t)max_targets * 4, ctx->stream));
  CK(cudaMemsetAsync(db->dL.p, 0, (size_t)max_targets * 4, ctx->stream));
  CK(cudaMemsetAsync(db->dcol_off.p, 0, (size_t)max_targets * 8, ctx->stream));
  CK(cudaMemsetAsync(db->pav.p, 0, (size_t)max_targets * 80, ctx->stream));
  CK(cudaMemsetAsync(db->cols_raw.p, 0, (size_t)max_cols * sizeof(ColRec), ctx->stream));
  CK(cudaMemsetAsync(db->cols.p, 0, (size_t)max_cols * sizeof(ColRec), ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  db->stage.reset(new StageCache(max_targets, max_cols));
  *out = std::move(db);
  return HHG_OK;
}

int hhg_db_create_staged(hhg_ctx* ctx, hhg_dbstore* store, int max_targets, long long max_cols, hhg_db** out) {
  if (!ctx || !store || !out || max_targets < 1 || max_cols < 1) return fail(HHG_EINVAL, "hhg_db_create_staged: bad argument");
  if (store->device != ctx->device)
    return fail(HHG_EINVAL, "hhg_db_create_staged: the store is mapped for device %d, ctx is on %d", store->device, ctx->device);
  std::unique_ptr<hhg_db> db;
  int rc = staged_new(ctx, max_targets, max_cols, store->has_ss, &db);
  if (rc != HHG_OK) return rc;
  db->store = store;
  store->users++;
  *out = db.release();
  return HHG_OK;
}

// CTAs of k_stage_gather: 8 warps each with 3.5 KB of loads in flight; 32 CTAs hold ~0.9 MB, several times the
// bandwidth-delay product of a PCIe 5 x16 link (DESIGN 4.12 has the sweep).  HHG_STAGE_CTAS: developer knob of that sweep.
static int stage_ctas() {
  const char* e = getenv("HHG_STAGE_CTAS");
  const int x = e ? atoi(e) : 0;
  return x > 0 ? x : 32;
}

template <class B>
static int stage_records(hhg_ctx* ctx, hhg_db* db, B& b, int n, const int32_t* ids, int32_t* local_out,
                         hhg_stage_stats* stats_out);

int hhg_db_stage(hhg_ctx* ctx, hhg_db* db, int n, const int32_t* global_ids, int32_t* local_ids_out,
                 hhg_stage_stats* stats_out) {
  if (!ctx || !db || n < 0 || (n && (!global_ids || !local_ids_out))) return fail(HHG_EINVAL, "hhg_db_stage: bad argument");
  if (!db->stage) return fail(HHG_EINVAL, "hhg_db_stage: the shard was not made by hhg_db_create_staged");
  if (db->device != ctx->device) return fail(HHG_EINVAL, "db lives on device %d, ctx on %d", db->device, ctx->device);
  if (db->src) {
    if (db->src->kind == 0) return stage_records(ctx, db, *std::static_pointer_cast<HhmBuilder>(db->builder), n, global_ids, local_ids_out, stats_out);
    return stage_records(ctx, db, *std::static_pointer_cast<MsaBuilder>(db->builder), n, global_ids, local_ids_out, stats_out);
  }
  const hhg_dbstore* st = db->store;
  std::vector<StageItem> items;
  std::vector<int> freed;
  StageStats ss{};
  int bad = 0;
  long long need_slots = 0, need_cols = 0;
  const int rc = db->stage->request(n, global_ids, st->n, st->L.data(), st->col_off.data(), local_ids_out, &items, &freed,
                                    &ss, &bad, &need_slots, &need_cols);
  if (rc == -1) return fail(HHG_EINVAL, "hhg_db_stage: request %d: target id %d outside the store (%d targets)", bad, global_ids[bad], st->n);
  if (rc == -2)
    return fail(HHG_EINVAL, "hhg_db_stage: the request needs %lld slots and %lld columns, the staged shard has %d and %lld",
                need_slots, need_cols, db->n, db->total_cols);
  static_assert(sizeof(hhg_stage_stats) == sizeof(StageStats), "hhg_stage_stats layout");
  if (stats_out) memcpy(stats_out, &ss, sizeof ss);
  if (items.empty() && freed.empty()) return HHG_OK;
  // one descriptor per copied target, then one per slot that only lost its target; run0 = first work item
  std::vector<StageDesc> desc;
  desc.reserve(items.size() + freed.size());
  long long runs = 0;
  for (const StageItem& it : items) {
    desc.push_back(StageDesc{it.src, it.dst, it.len, it.slot, it.global, (int)runs});
    runs += (it.len + kStageRun - 1) / kStageRun;
    db->L[it.slot] = it.len;
    db->col_off[it.slot] = it.dst;
  }
  for (int s : freed) {
    desc.push_back(StageDesc{0, 0, 0, s, 0, (int)runs});
    db->L[s] = 0;
  }
  // every plan over this shard describes the old slots: a new identity makes plan_build start over and hhg_plan_run
  // refuse; `cols` no longer holds the null model of the new records
  db->serial = g_db_serial.fetch_add(1);
  db->cols_version++;
  db->prepared = false;
  CK(cudaSetDevice(ctx->device));
  int arc = ctx_aux_stream(ctx);
  if (arc != HHG_OK) return arc;
  CK(db->d_desc.ensure(desc.size()));
  // work already queued on the context stream may read the records this call overwrites, and may still read the
  // descriptor buffer's last content: the gather starts after it, and the context stream goes on after the gather
  CK(cudaEventRecord(ctx->aux_ev[0], ctx->stream));
  CK(cudaStreamWaitEvent(ctx->aux_stream, ctx->aux_ev[0], 0));
  CK(cudaMemcpyAsync(db->d_desc.p, desc.data(), desc.size() * sizeof(StageDesc), cudaMemcpyHostToDevice, ctx->aux_stream));
  const int ctas = (int)std::max(1LL, std::min<long long>(stage_ctas(), std::max<long long>((runs + 7) / 8, ((long long)desc.size() + 31) / 32)));
  k_stage_gather<<<ctas, 256, 0, ctx->aux_stream>>>((int)desc.size(), (int)runs, db->d_desc.p, st->d_cols, st->d_pav,
                                                    db->cols_raw.p, db->pav.p, db->dL.p, db->dcol_off.p);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->aux_ev[1], ctx->aux_stream));
  CK(cudaStreamWaitEvent(ctx->stream, ctx->aux_ev[1], 0));
  return HHG_OK;
}

int hhg_db_staged_lookup(const hhg_db* db, int n, const int32_t* local_ids, int32_t* global_ids_out, int64_t* first_col_out) {
  if (!db || !db->stage || n < 0 || (n && !local_ids)) return fail(HHG_EINVAL, "hhg_db_staged_lookup: bad argument / shard not staged");
  for (int k = 0; k < n; ++k) {
    const int s = local_ids[k];
    if (s < 0 || s >= db->n) return fail(HHG_EINVAL, "hhg_db_staged_lookup: local id %d out of range", s);
    if (global_ids_out) global_ids_out[k] = db->stage->global_of(s);
    if (first_col_out) first_col_out[k] = db->stage->off_of(s);
  }
  return HHG_OK;
}

// ------------------------------------------------------------------------- record source + staged shard over it
// What prefilter_db + HHEntry::getTemplateHMM do (src/hhprefilter.cpp:561-590, src/hhdatabase.cpp:300-336,
// :398-461): only the survivors' records are ever parsed, when hhg_db_stage makes them resident (DESIGN 4.12).
static int recsrc_new(hhg_ctx* ctx, const char* who, int kind, int n, const char* data, const int64_t* off,
                      const int64_t* len, const hhg_seqdb* seqs, const hhg_msa_params* mp, const float* S,
                      const float* pb, const hhg_prep_params* pp, const float* R, int has_ss, hhg_recsrc** out) {
  if (!ctx || !out || n < 1 || !data || !off || !len || !pp || !R || (kind && !pb))
    return fail(HHG_EINVAL, "%s: bad argument", who);
  HhmPrepArgs A;
  int rc = kind ? msa_load_args(who, seqs, mp, S, pp, R, &A) : hhm_prep_args(who, pp, R, &A);
  if (rc != HHG_OK) return rc;
  for (int k = 0; k < n; ++k)
    if (off[k] < 0 || len[k] < 0) return fail(HHG_EINVAL, "%s: record %d: offset %lld, length %lld", who, k, (long long)off[k], (long long)len[k]);
  std::unique_ptr<hhg_recsrc> src(new hhg_recsrc());
  src->device = ctx->device;
  src->kind = kind;
  src->n = n;
  src->data = data;
  src->off.assign(off, off + n);
  src->len.assign(len, len + n);
  if (seqs) src->seqs = *seqs;
  if (mp) src->mp = *mp;
  src->pp = *pp;
  if (S) src->S.assign(S, S + 400);
  if (pb) src->pb.assign(pb, pb + 20);
  src->R.assign(R, R + 400);
  src->has_ss = has_ss != 0;
  src->L.assign(n, 0);
  *out = src.release();
  return HHG_OK;
}

int hhg_recsrc_create_hhm(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                          const hhg_prep_params* pp, const float* R, int has_ss, hhg_recsrc** out) {
  return recsrc_new(ctx, "hhg_recsrc_create_hhm", 0, n, data, off, len, nullptr, nullptr, nullptr, nullptr, pp, R, has_ss, out);
}

int hhg_recsrc_create_a3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                          const hhg_msa_params* mp, const float* S, const float* pb, const hhg_prep_params* pp,
                          const float* R, int has_ss, hhg_recsrc** out) {
  return recsrc_new(ctx, "hhg_recsrc_create_a3m", 1, n, data, off, len, nullptr, mp, S, pb, pp, R, has_ss, out);
}

int hhg_recsrc_create_ca3m(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len,
                           const hhg_seqdb* seqs, const hhg_msa_params* mp, const float* S, const float* pb,
                           const hhg_prep_params* pp, const float* R, int has_ss, hhg_recsrc** out) {
  if (!seqs) return fail(HHG_EINVAL, "hhg_recsrc_create_ca3m: the sequence database is NULL");
  return recsrc_new(ctx, "hhg_recsrc_create_ca3m", 2, n, data, off, len, seqs, mp, S, pb, pp, R, has_ss, out);
}

int hhg_recsrc_destroy(hhg_recsrc* src) {
  if (!src) return HHG_OK;
  if (src->users > 0) return fail(HHG_EINVAL, "hhg_recsrc_destroy: %d staged shards still use the record source", src->users);
  delete src;
  return HHG_OK;
}

int hhg_recsrc_size(const hhg_recsrc* src) { return src ? src->n : 0; }

int hhg_db_create_staged_records(hhg_ctx* ctx, hhg_recsrc* src, int max_targets, long long max_cols, hhg_db** out) {
  if (!ctx || !src || !out || max_targets < 1 || max_cols < 1) return fail(HHG_EINVAL, "hhg_db_create_staged_records: bad argument");
  if (src->device != ctx->device)
    return fail(HHG_EINVAL, "hhg_db_create_staged_records: the record source was made for device %d, ctx is on %d", src->device, ctx->device);
  std::unique_ptr<hhg_db> db;
  int rc = staged_new(ctx, max_targets, max_cols, src->has_ss, &db);
  if (rc != HHG_OK) return rc;
  const RecText T{src->data, src->off.data(), src->len.data()};
  if (src->kind == 0) {
    auto b = std::make_shared<HhmBuilder>();
    b->T = T; b->pp = &src->pp;
    if ((rc = hhm_prep_args("hhg_db_create_staged_records", &src->pp, src->R.data(), &b->A)) != HHG_OK) return rc;
    db->builder = b;
  } else {
    auto b = std::make_shared<MsaBuilder>();
    b->T = T; b->sq = src->kind == 2 ? &src->seqs : nullptr; b->mp = &src->mp;
    b->S = src->S.empty() ? nullptr : src->S.data(); b->pb = src->pb.data(); b->pp = &src->pp;
    if ((rc = hhm_prep_args("hhg_db_create_staged_records", &src->pp, src->R.data(), &b->A)) != HHG_OK) return rc;
    db->builder = b;
  }
  db->neff.assign(max_targets, 0.f);
  db->src = src;
  src->users++;
  *out = db.release();
  return HHG_OK;
}

// The error just recorded, prefixed with the entry point's name.
static int stage_error(int rc) {
  const std::string msg = hhg_last_error();
  return fail(rc, "hhg_db_stage: %s", msg.c_str());
}

// After a failure between the placement and the last gather the slot tables no longer describe the arena: every
// slot is emptied (a new identity, as for any call that changes a slot).
static void stage_clear(hhg_ctx* ctx, hhg_db* db) {
  db->stage.reset(new StageCache(db->n, db->total_cols));
  std::fill(db->L.begin(), db->L.end(), 0);
  std::fill(db->col_off.begin(), db->col_off.end(), 0);
  std::fill(db->neff.begin(), db->neff.end(), 0.f);
  cudaMemsetAsync(db->dL.p, 0, (size_t)db->n * 4, ctx->stream);
  cudaStreamSynchronize(ctx->stream);
  db->serial = g_db_serial.fetch_add(1);
  db->cols_version++;
  db->prepared = false;
}

// hhg_db_stage on a record-sourced shard: the request's missing records are scanned on the host threads (their lengths
// and every parse error before anything changes), StageCache places them exactly as it places a store's targets, and
// the targets to copy are built in groups by the loaders' builder into rec_cols / rec_pav, from where k_stage_gather
// moves them into their arena runs.  A re-layout of the request's own residents rebuilds them from their records.
// The host is blocked for the scan and the build.
template <class B>
static int stage_records(hhg_ctx* ctx, hhg_db* db, B& b, int n, const int32_t* ids, int32_t* local_out,
                         hhg_stage_stats* stats_out) {
  hhg_recsrc* src = db->src;
  CK(cudaSetDevice(ctx->device));
  b.ctx = ctx;
  const bool timing = getenv("HHG_TIMING") != nullptr;
  const auto t_begin = std::chrono::steady_clock::now();
  // 1. the distinct missing records, in the order StageCache will place them
  std::vector<int32_t> miss;
  {
    std::unordered_set<int> seen;
    for (int k = 0; k < n; ++k) {
      const int g = ids[k];
      if (g < 0 || g >= src->n)
        return fail(HHG_EINVAL, "hhg_db_stage: request %d: target id %d outside the record source (%d records)", k, g, src->n);
      if (db->stage->slot_of(g) < 0 && seen.insert(g).second) miss.push_back(g);
    }
  }
  // 2-3. their lengths: LENG lines of HHM records (peek), then the full parse of every group, which also refuses a
  // malformed alignment; the parse of the last group stays in b and is used again below when it is what gets built
  const int nm = (int)miss.size();
  std::vector<int32_t> Lm(nm);
  int rc = b.peek(miss.data(), nm, Lm.data());
  if (rc != HHG_OK) return stage_error(rc);
  if (std::is_same<B, HhmBuilder>::value) {
    for (int k = 0; k < nm; ++k)
      if (Lm[k] < 1 || Lm[k] > 32767) return fail(HHG_EINVAL, "hhg_db_stage: record %d: length %d out of [1,32767]", miss[k], Lm[k]);
    for (int k = 0; k < nm; ++k) src->L[miss[k]] = Lm[k];
  }
  for (int k0 = 0, k1; k0 < nm; k0 = k1) {
    k1 = b.group_end(miss.data(), k0, nm, src->L.data());
    if ((rc = b.scan(miss.data() + k0, k1 - k0)) != HHG_OK) return stage_error(rc);
    for (int k = 0; k < k1 - k0; ++k) src->L[b.rec[k]] = b.L[k];
  }
  const double ms_scan = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
  // 4. placement (the record offsets stand in for store offsets: every item's source is replaced below)
  static_assert(sizeof(int64_t) == sizeof(long long), "record offsets as StageCache source offsets");
  std::vector<StageItem> items;
  std::vector<int> freed;
  StageStats ss{};
  int bad = 0;
  long long need_slots = 0, need_cols = 0;
  rc = db->stage->request(n, ids, src->n, src->L.data(), reinterpret_cast<const long long*>(src->off.data()), local_out,
                          &items, &freed, &ss, &bad, &need_slots, &need_cols);
  if (rc == -1) return fail(HHG_EINVAL, "hhg_db_stage: request %d: target id %d outside the record source (%d records)", bad, ids[bad], src->n);
  if (rc == -2)
    return fail(HHG_EINVAL, "hhg_db_stage: the request needs %lld slots and %lld columns, the staged shard has %d and %lld",
                need_slots, need_cols, db->n, db->total_cols);
  if (stats_out) memcpy(stats_out, &ss, sizeof ss);
  if (items.empty() && freed.empty()) return HHG_OK;
  for (const StageItem& it : items) { db->L[it.slot] = it.len; db->col_off[it.slot] = it.dst; }
  for (int s : freed) db->L[s] = 0;
  db->serial = g_db_serial.fetch_add(1);
  db->cols_version++;
  db->prepared = false;
  // 5-6. build the copied targets group by group, each group gathered from the scratch into its arena runs; descriptor
  // k of a group reads scratch records from the builder's rec_off[k] and pav row k
  const int ni = (int)items.size();
  std::vector<int32_t> order(ni);
  for (int k = 0; k < ni; ++k) order[k] = items[k].global;
  std::vector<StageDesc> desc;
  std::vector<float> neff;
  double ms_build = 0.0, ms_gather = 0.0;
  for (int k0 = 0, k1; k0 < ni; k0 = k1) {
    const auto t0 = std::chrono::steady_clock::now();
    k1 = b.group_end(order.data(), k0, ni, src->L.data());
    const int m = k1 - k0;
    if (!((int)b.rec.size() == m && std::equal(b.rec.begin(), b.rec.end(), order.begin() + k0)) &&
        (rc = b.scan(order.data() + k0, m)) != HHG_OK) {
      stage_clear(ctx, db);
      return stage_error(rc);
    }
    neff.resize(m);
    cudaError_t e = db->rec_cols.ensure((size_t)b.cols * 7);
    if (e == cudaSuccess) e = db->rec_pav.ensure((size_t)m * 20);
    rc = e == cudaSuccess ? b.build(src->has_ss, reinterpret_cast<ColRec*>(db->rec_cols.p), db->rec_pav.p, nullptr, neff.data())
                          : fail(HHG_ECUDA, "%s", cudaGetErrorString(e));
    if (rc != HHG_OK) { stage_clear(ctx, db); return stage_error(rc); }
    const auto t1 = std::chrono::steady_clock::now();
    ms_build += std::chrono::duration<double, std::milli>(t1 - t0).count();
    desc.clear();
    long long runs = 0;
    for (int k = 0; k < m; ++k) {
      const StageItem& it = items[k0 + k];
      desc.push_back(StageDesc{b.rec_off[k], it.dst, it.len, it.slot, k, (int)runs});
      runs += (it.len + kStageRun - 1) / kStageRun;
      db->neff[it.slot] = neff[k];
    }
    if (k0 == 0)
      for (int s : freed) desc.push_back(StageDesc{0, 0, 0, s, 0, (int)runs});
    e = db->d_desc.ensure(desc.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(db->d_desc.p, desc.data(), desc.size() * sizeof(StageDesc), cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess) {
      const int ctas = (int)std::max(1LL, std::min<long long>(stage_ctas(), std::max<long long>((runs + 7) / 8, ((long long)desc.size() + 31) / 32)));
      k_stage_gather<<<ctas, 256, 0, ctx->stream>>>((int)desc.size(), (int)runs, db->d_desc.p, db->rec_cols.p, db->rec_pav.p,
                                                    db->cols_raw.p, db->pav.p, db->dL.p, db->dcol_off.p);
      ctx->launches++;
      e = cudaGetLastError();
    }
    if (e == cudaSuccess && timing) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { stage_clear(ctx, db); return fail(HHG_ECUDA, "hhg_db_stage: %s", cudaGetErrorString(e)); }
    ms_gather += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t1).count();
  }
  if (timing)
    fprintf(stderr, "[hhg] record stage: %d missing records, %d built, host scan %.3f ms, build %.3f ms, gather %.3f ms\n",
            nm, ni, ms_scan, ms_build, ms_gather);
  return HHG_OK;
}

int hhg_db_staged_neff(const hhg_db* db, int n, const int32_t* local_ids, float* neff_out) {
  if (!db || !db->stage || n < 0 || (n && (!local_ids || !neff_out))) return fail(HHG_EINVAL, "hhg_db_staged_neff: bad argument / shard not staged");
  if (!db->src) return fail(HHG_EINVAL, "hhg_db_staged_neff: the shard stages from a store of packed records, which holds no Neff");
  for (int k = 0; k < n; ++k) {
    const int s = local_ids[k];
    if (s < 0 || s >= db->n) return fail(HHG_EINVAL, "hhg_db_staged_neff: local id %d out of range", s);
    if (db->L[s] < 1) return fail(HHG_EINVAL, "hhg_db_staged_neff: slot %d of the staged shard is empty", s);
    neff_out[k] = db->neff[s];
  }
  return HHG_OK;
}

// --------------------------------------------------------------------------------------- query
static int query_set_impl(hhg_ctx* ctx, int nq, const int32_t* Lq, const float* const* p, const float* const* tr,
                          const uint8_t* const* ss, const float* q_pav, const float* S33, const hhg_params* par) {
  if (!ctx || nq < 1 || !Lq || !p || !tr || !par) return fail(HHG_EINVAL, "hhg_query_set: bad argument");
  bool all_ss = ss != nullptr;
  for (int q = 0; q < nq; ++q) {
    if (Lq[q] < 1 || Lq[q] > 32767 || !p[q] || !tr[q]) return fail(HHG_EINVAL, "hhg_query_set: bad query %d", q);
    if (ss && !ss[q]) all_ss = false;
  }
  if (par->use_ss && (!all_ss || !S33)) return fail(HHG_EINVAL, "hhg_query_set: use_ss needs ss and S33");
  CK(cudaSetDevice(ctx->device));
  ctx->par = *par;
  ctx->nq = nq;
  ctx->q_L.assign(Lq, Lq + nq);
  ctx->q_row0.resize(nq);
  long long rows = 0;
  for (int q = 0; q < nq; ++q) {
    ctx->q_row0[q] = (int)rows;
    rows += (Lq[q] + 47) / 48 * 48;     // each query zero padded to a multiple of every strip height (8, 12, 16)
  }
  if (rows > 0x7fffffffLL / 7) return fail(HHG_EINVAL, "hhg_query_set: query batch too large");
  ctx->Lq = Lq[0];
  CK(ctx->qrec.ensure((size_t)rows * 7));
  CK(cudaMemsetAsync(ctx->qrec.p, 0, (size_t)rows * 112, ctx->stream));
  // pack with the same kernel as the DB (one-profile shards)
  for (int q = 0; q < nq; ++q) {
    std::vector<long long> col_off(1, 0);
    const int32_t L1 = Lq[q];
    const int64_t zero = 0;
    int rc = pack_profiles(ctx, 1, &L1, &zero, &zero, &zero, p[q], tr[q], ss ? ss[q] : nullptr, col_off, L1,
                           ctx->qrec.p + (size_t)ctx->q_row0[q] * 7);
    if (rc != HHG_OK) return rc;
  }
  ctx->has_ss = all_ss;
  ctx->has_S33 = false;
  if (S33) {
    CK(ctx->S33.ensure(44 * 44));
    CK(cudaMemcpyAsync(ctx->S33.p, S33, 44 * 44 * 4, cudaMemcpyHostToDevice, ctx->stream));
    ctx->has_S33 = true;
  }
  ctx->has_q_pav = q_pav != nullptr;
  if (q_pav) {
    ctx->h_q_pav.assign(q_pav, q_pav + (size_t)nq * 20);
    CK(ctx->d_q_pav.ensure((size_t)nq * 20));
    CK(cudaMemcpyAsync(ctx->d_q_pav.p, q_pav, (size_t)nq * 80, cudaMemcpyHostToDevice, ctx->stream));
  }
  ctx->query_serial++;
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

int hhg_query_set(hhg_ctx* ctx, int Lq, const float* p, const float* tr, const uint8_t* ss,
                  const float* S33, const hhg_params* par) {
  const int32_t L1 = Lq;
  return query_set_impl(ctx, 1, &L1, &p, &tr, ss ? &ss : nullptr, nullptr, S33, par);
}

int hhg_query_set_batch(hhg_ctx* ctx, int nq, const int32_t* Lq, const float* const* p, const float* const* tr,
                        const uint8_t* const* ss, const float* q_pav, const float* S33, const hhg_params* par) {
  return query_set_impl(ctx, nq, Lq, p, tr, ss, q_pav, S33, par);
}

// Switch the PRED_PRED secondary-structure term on/off for the following searches without re-sending the query
// (Viterbi::Align picks the *AndSS kernels per 8-target batch, src/hhviterbirunner.cpp:14-26).
int hhg_set_use_ss(hhg_ctx* ctx, int use_ss) {
  if (!ctx) return fail(HHG_EINVAL, "ctx is NULL");
  if (use_ss && (!ctx->has_ss || !ctx->has_S33)) return fail(HHG_EINVAL, "hhg_set_use_ss: the query was set without ss / S33");
  ctx->par.use_ss = use_ss ? 1 : 0;
  return HHG_OK;
}

// ---------------------------------------------------------------------------------------- plan
// Strip height of a plan.  Whole-shard scans have work items to spare and take R = 16: the least per-column overhead
// (boundary hand-off, operand copies, running maximum) per row.  R = 12 fits 3 CTAs per SM instead of 2 but measures
// slower on an H100 (400 W limit, SM clock 1.59-1.64 GHz): 61.8-62.8 ms against 55.6-55.8 ms per launch at Lq = 400
// (34 strips of 12, 2 % padded rows) and 55.9-56.2 against 55.5-55.7 ms at Lq = 1500 (tools/vit_ab.py).
// A small request (the few thousand survivors of the prefilter) is latency bound: its longest job is one serial sweep
// over Lmax columns per strip, so halving the strip height halves that critical path and doubles the number of work
// items that can run side by side.
static int plan_strip_rows(const hhg_ctx* ctx, const int32_t* req_query, int n) {
  if (ctx->R) return ctx->R;
  long long items16 = 0;
  if (!req_query) items16 = (long long)((n + 31) / 32) * ((ctx->q_L[0] + 15) / 16);
  else {
    std::vector<long long> cnt(ctx->nq, 0);
    for (int k = 0; k < n; ++k) if (req_query[k] >= 0 && req_query[k] < ctx->nq) cnt[req_query[k]]++;
    for (int q = 0; q < ctx->nq; ++q) items16 += (cnt[q] + 31) / 32 * ((ctx->q_L[q] + 15) / 16);
  }
  return items16 >= 4LL * ctx->sm_count * 8 ? 16 : 8;
}

// (Re)build a plan in place; device buffers only ever grow, so a plan object that is reused across
// searches (hhg_viterbi_search keeps one per context) does not touch cudaMalloc in steady state.
// req_query[k] = index (into the context's query batch) of the query request k is aligned with; NULL = query 0.
// Jobs never mix queries: the requests of each query are length-sorted and cut into 32-target jobs separately.
static int plan_build(hhg_ctx* ctx, hhg_plan* pl, const hhg_db* db, int n, const int32_t* ids,
                      const int32_t* req_query = nullptr) {
  if (!ctx || !db || n <= 0) return fail(HHG_EINVAL, "hhg_plan_create: bad argument");
  if (ctx->nq <= 0) return fail(HHG_EINVAL, "hhg_plan_create: no query set");
  if (db->device != ctx->device) return fail(HHG_EINVAL, "db lives on device %d, ctx on %d", db->device, ctx->device);
  CK(cudaSetDevice(ctx->device));
  const int R = plan_strip_rows(ctx, req_query, n);
  // the common case of a repeated request (same shard, same target list, same query batch geometry, e.g. every
  // query of a series against the whole shard) reuses the plan: no host sort, no uploads
  if (pl->built && pl->db == db && pl->db_serial == db->serial && pl->n == n && pl->R == R && pl->q_L == ctx->q_L &&
      pl->q_row0 == ctx->q_row0 && !pl->ids.empty() && pl->max_bt_bytes == ctx->max_bt_bytes) {
    bool same = true;
    if (ids) same = memcmp(ids, pl->ids.data(), (size_t)n * 4) == 0;
    else for (int k = 0; k < n && same; ++k) same = pl->ids[k] == k;
    if (same) {
      if (req_query) same = memcmp(req_query, pl->req_query.data(), (size_t)n * 4) == 0;
      else for (int k = 0; k < n && same; ++k) same = pl->req_query[k] == 0;
    }
    if (same) { pl->celloff = false; return HHG_OK; }
  }
  // any early return below leaves the plan half rewritten: it must neither be reused nor run until a build succeeds
  pl->built = false;
  pl->db = db;
  pl->db_serial = db->serial;
  pl->device = db->device;
  pl->max_bt_bytes = ctx->max_bt_bytes;
  pl->cells = pl->padded_cells = pl->alg_bytes = 0;
  pl->waves.clear();
  pl->celloff = false;
  pl->n = n;
  pl->R = R;
  pl->q_L = ctx->q_L; pl->q_row0 = ctx->q_row0;
  pl->Lq = ctx->q_L[0];
  pl->ids.resize(n); pl->req_query.resize(n);
  for (int k = 0; k < n; ++k) {
    const int id = ids ? ids[k] : k;
    if (id < 0 || id >= db->n) return fail(HHG_EINVAL, "request %d: target id %d out of range", k, id);
    if (db->L[id] < 1) return fail(HHG_EINVAL, "request %d: slot %d of the staged shard is empty", k, id);
    const int q = req_query ? req_query[k] : 0;
    if (q < 0 || q >= ctx->nq) return fail(HHG_EINVAL, "request %d: query index %d out of range (batch of %d)", k, q, ctx->nq);
    pl->ids[k] = id; pl->req_query[k] = q;
  }
  // sort requests by (query, target length descending) (the length sort is what ViterbiRunner does per chunk,
  // src/hhviterbirunner.cpp:117-119; here it also makes LPT scheduling of the work queue)
  pl->order.resize(n);
  std::iota(pl->order.begin(), pl->order.end(), 0);
  std::stable_sort(pl->order.begin(), pl->order.end(), [&](int a, int b) {
    if (pl->req_query[a] != pl->req_query[b]) return pl->req_query[a] < pl->req_query[b];
    return db->L[pl->ids[a]] > db->L[pl->ids[b]];
  });
  // jobs: runs of up to 32 consecutive sorted requests of the same query
  pl->jobs.clear();
  pl->reqs.assign(n, ReqDesc{});
  pl->jc_version = 0;
  std::vector<int> job_target;
  long long bnd = 0, co = 0, jc = 0, ss = 0;
  size_t wave_bt = 0, max_wave_words = 0;   // words in the current wave
  Wave w;
  for (int first = 0; first < n;) {
    const int jb = (int)pl->jobs.size();
    const int q = pl->req_query[pl->order[first]];
    int cnt = 0;
    while (first + cnt < n && cnt < 32 && pl->req_query[pl->order[first + cnt]] == q) ++cnt;
    const int Lmax = db->L[pl->ids[pl->order[first]]];
    const int ns = (ctx->q_L[q] + R - 1) / R;
    for (int l = 0; l < 32; ++l) {
      const int rq = pl->order[first + std::min(l, cnt - 1)];   // padded lanes repeat the last target
      job_target.push_back(pl->ids[rq]);
      if (l < cnt) { pl->reqs[rq].job = jb; pl->reqs[rq].lane = l; }
    }
    const size_t words = (size_t)(ns * R / 4) * (Lmax + 1) * 32;
    if (wave_bt > 0 && (wave_bt + words) * 4 > ctx->max_bt_bytes) {
      w.job_end = jb;
      pl->waves.push_back(w);
      max_wave_words = std::max(max_wave_words, wave_bt);
      w.job_begin = jb;
      wave_bt = 0;
    }
    JobDesc d{};
    d.ss_off = ss; d.bt_off = (long long)wave_bt; d.bnd_off = bnd; d.co_off = co; d.jc_off = jc;
    d.Lmax = Lmax; d.query = q; d.nstrips = ns; d.Lq = ctx->q_L[q]; d.qrow0 = ctx->q_row0[q];
    pl->jobs.push_back(d);
    wave_bt += words;
    bnd += (long long)(Lmax + 1) * 32;
    jc += (long long)Lmax * 224;
    co += (long long)ns * (Lmax + 1) * 32;
    ss += ns;
    pl->padded_cells += (double)ns * R * (double)Lmax * 32.0;
    first += cnt;
  }
  pl->njobs = (int)pl->jobs.size();
  w.job_end = pl->njobs;
  pl->waves.push_back(w);
  max_wave_words = std::max(max_wave_words, wave_bt);
  pl->ss_total = ss;
  pl->co_total = co;
  // work items (job, strip) of every wave in dispatch order: groups of G consecutive jobs, strip-major inside a group
  // (strip s of all the group's jobs, then strip s+1, ...), so consecutive strips of a job are G items apart
  pl->items.clear();
  for (Wave& wv : pl->waves) {
    wv.item_begin = (long long)pl->items.size();
    for (int g0 = wv.job_begin; g0 < wv.job_end; g0 += ctx->group_jobs) {
      const int g1 = std::min(g0 + ctx->group_jobs, wv.job_end);
      int maxns = 0;
      for (int jb = g0; jb < g1; ++jb) maxns = std::max(maxns, pl->jobs[jb].nstrips);
      for (int sidx = 0; sidx < maxns; ++sidx)
        for (int jb = g0; jb < g1; ++jb)
          if (sidx < pl->jobs[jb].nstrips) pl->items.push_back(make_int2(jb - wv.job_begin, sidx));
    }
    wv.item_end = (long long)pl->items.size();
  }
  long long po = 0;
  double cols_sum = 0;
  for (int k = 0; k < n; ++k) {
    ReqDesc& r = pl->reqs[k];
    r.target = pl->ids[k];
    r.Lt = db->L[r.target];
    r.Lq = ctx->q_L[pl->req_query[k]];
    r.path_off = po;
    po += r.Lq + r.Lt + 2;
    pl->cells += (double)r.Lq * r.Lt;
    cols_sum += r.Lt;
  }
  if (po > 0x7fffffffLL) return fail(HHG_EINVAL, "plan too large: %lld path bytes (> 2^31-1); split the request", po);
  pl->path_total = po;
  pl->jc_total = jc;
  pl->alg_bytes = cols_sum * 112.0 + pl->cells * 1.0 + (double)sizeof(HitRec) * n;

  cudaError_t e = cudaSuccess;
  auto A = [&](cudaError_t r) { if (e == cudaSuccess) e = r; };
  A(pl->d_jobs.ensure(pl->njobs)); A(pl->d_reqs.ensure(n));
  A(pl->d_job_target.ensure(job_target.size())); A(pl->d_items.ensure(pl->items.size()));
  // one column (224 float4) and one slot column (32 slots) of slack: k_viterbi prefetches column j+1 unconditionally,
  // so at the last job's last column it reads one column past the operand stream and the slots (never used)
  A(pl->d_jcols.ensure((size_t)jc + 224));
  A(pl->d_S.ensure((size_t)po));
  A(pl->d_bt.ensure(max_wave_words));
  { BndSlot* before = pl->d_bnd.p; A(pl->d_bnd.ensure((size_t)bnd + 32));
    // fresh slots must not carry a bit pattern that looks like a valid tag (epochs start at 1)
    if (e == cudaSuccess && pl->d_bnd.p != before) A(cudaMemsetAsync(pl->d_bnd.p, 0, pl->d_bnd.n * sizeof(BndSlot), ctx->stream)); }
  A(pl->d_strip_score.ensure((size_t)ss * 32));
  A(pl->d_strip_ij.ensure((size_t)ss * 32));
  A(pl->d_counter.ensure(pl->waves.size()));
  A(pl->d_hits.ensure(n));
  A(pl->d_paths.ensure((size_t)po));
  if (e != cudaSuccess) return fail(HHG_ENOMEM, "hhg_plan_create: %s", cudaGetErrorString(e));

  cudaStream_t st = ctx->stream;
  auto H2D = [&](void* d, const void* h, size_t bytes) { return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st); };
  CK(H2D(pl->d_jobs.p, pl->jobs.data(), pl->jobs.size() * sizeof(JobDesc)));
  CK(H2D(pl->d_reqs.p, pl->reqs.data(), pl->reqs.size() * sizeof(ReqDesc)));
  CK(H2D(pl->d_job_target.p, job_target.data(), job_target.size() * 4));
  CK(H2D(pl->d_items.p, pl->items.data(), pl->items.size() * sizeof(int2)));
  CK(cudaStreamSynchronize(st));
  pl->built = true;
  return HHG_OK;
}

int hhg_plan_create(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* ids, hhg_plan** out) {
  if (!out) return fail(HHG_EINVAL, "hhg_plan_create: out is NULL");
  std::unique_ptr<hhg_plan> pl(new hhg_plan());
  int rc = plan_build(ctx, pl.get(), db, n, ids);
  if (rc != HHG_OK) return rc;
  *out = pl.release();
  return HHG_OK;
}

int hhg_plan_destroy(hhg_plan* plan) {
  if (plan) { if (plan->db) cudaSetDevice(plan->device); delete plan; }
  return HHG_OK;
}
double hhg_plan_cells(const hhg_plan* plan) { return plan ? plan->cells : 0; }
double hhg_plan_padded_cells(const hhg_plan* plan) { return plan ? plan->padded_cells : 0; }
double hhg_plan_algorithmic_bytes(const hhg_plan* plan) { return plan ? plan->alg_bytes : 0; }

// the context's excluded regions into ctx->d_ex, on ctx->stream
static int upload_regions(hhg_ctx* ctx) {
  CK(ctx->d_ex.ensure(ctx->ex.size()));
  CK(cudaMemcpyAsync(ctx->d_ex.p, ctx->ex.data(), ctx->ex.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  return HHG_OK;
}

static int set_exclusions(hhg_ctx* ctx, hhg_plan* pl, const int64_t* excl_off, const int32_t* excl_i,
                          const int32_t* excl_j) {
  pl->celloff = false;
  pl->n_excl_steps = 0;
  const long long total = excl_off ? excl_off[pl->n] : 0;
  const bool regions = !ctx->ex.empty();
  if (total <= 0 && !regions) return HHG_OK;
  const size_t co_words = (size_t)pl->co_total;
  CK(pl->d_co.ensure(co_words));
  CK(cudaMemsetAsync(pl->d_co.p, 0, co_words * 4, ctx->stream));
  if (total > 0) {
    // validate like hhg_mac_realign does: k_celloff_raster indexes the mask with these values
    if (excl_off[0] != 0) return fail(HHG_EINVAL, "excl_off[0] must be 0");
    if (!excl_i || !excl_j) return fail(HHG_EINVAL, "excl_i / excl_j are NULL");
    std::vector<int> sreq((size_t)total);
    for (int k = 0; k < pl->n; ++k) {
      if (excl_off[k + 1] < excl_off[k]) return fail(HHG_EINVAL, "excl_off is not monotonic at request %d", k);
      const int Lt = pl->reqs[k].Lt, Lqk = pl->reqs[k].Lq;
      for (long long s = excl_off[k]; s < excl_off[k + 1]; ++s) {
        if (excl_i[s] < 1 || excl_i[s] > Lqk || excl_j[s] < 1 || excl_j[s] > Lt)
          return fail(HHG_EINVAL, "excluded step %lld of request %d is (%d,%d), outside 1..%d x 1..%d", s - excl_off[k], k,
                      excl_i[s], excl_j[s], Lqk, Lt);
        sreq[(size_t)s] = k;
      }
    }
    CK(pl->d_step_req.ensure((size_t)total)); CK(pl->d_step_i.ensure((size_t)total)); CK(pl->d_step_j.ensure((size_t)total));
    CK(cudaMemcpyAsync(pl->d_step_req.p, sreq.data(), (size_t)total * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(pl->d_step_i.p, excl_i, (size_t)total * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(pl->d_step_j.p, excl_j, (size_t)total * 4, cudaMemcpyHostToDevice, ctx->stream));
    const int threads = 128;
    k_celloff_raster<<<(unsigned)((total + threads - 1) / threads), threads, 0, ctx->stream>>>(
        (int)total, pl->d_step_req.p, pl->d_step_i.p, pl->d_step_j.p, pl->d_reqs.p, pl->d_jobs.p, pl->R, pl->d_co.p);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ctx->stream));   // sreq is a host temporary
  }
  if (regions) {
    const int nq = ctx->ex_nq, nt = ctx->ex_nt;
    const int rc = upload_regions(ctx);
    if (rc != HHG_OK) return rc;
    const int* d = ctx->d_ex.p;
    k_celloff_regions<<<(unsigned)((co_words + 255) / 256), 256, 0, ctx->stream>>>(
        (long long)co_words, pl->njobs, pl->d_jobs.p, pl->R, nq, d, d + nq, nt, d + 2 * nq, d + 2 * nq + nt, pl->d_co.p);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ctx->stream));
  }
  pl->celloff = true;
  pl->n_excl_steps = (int)total;
  return HHG_OK;
}

// -excl / -template_excl (par.exclstr / par.template_exclstr): ranges of query rows / template columns that are switched
// off in every following search of this context (ViterbiRunner::exclude_regions, src/hhviterbirunner.cpp:291-330);
// n = 0 clears.  Ranges are 1-based and inclusive like the option strings.
int hhg_set_excluded_regions(hhg_ctx* ctx, int nq, const int32_t* q_lo, const int32_t* q_hi, int nt, const int32_t* t_lo,
                             const int32_t* t_hi) {
  if (!ctx || nq < 0 || nt < 0 || (nq && (!q_lo || !q_hi)) || (nt && (!t_lo || !t_hi)))
    return fail(HHG_EINVAL, "hhg_set_excluded_regions: bad argument");
  ctx->ex.assign(q_lo, q_lo + nq);
  ctx->ex.insert(ctx->ex.end(), q_hi, q_hi + nq);
  ctx->ex.insert(ctx->ex.end(), t_lo, t_lo + nt);
  ctx->ex.insert(ctx->ex.end(), t_hi, t_hi + nt);
  ctx->ex_nq = nq;
  ctx->ex_nt = nt;
  return HHG_OK;
}

template <int R>
static int launch_viterbi(hhg_ctx* ctx, const VitParams& P, bool local, bool ss, bool co, int items) {
  // per warp: R query rows and the two-column operand ring; then the mbarriers and the S33 table
  const size_t smem = (size_t)kWarpsPerCta * (R * 112 + kRingBytes) + 64 + (ss ? 44 * 44 * 4 : 0);
  void (*kern)(const VitParams) = nullptr;
#define PICK(L_, S_, C_) kern = k_viterbi<R, L_, S_, C_>
  if (local) { if (ss) { if (co) PICK(true, true, true); else PICK(true, true, false); }
               else    { if (co) PICK(true, false, true); else PICK(true, false, false); } }
  else       { if (ss) { if (co) PICK(false, true, true); else PICK(false, true, false); }
               else    { if (co) PICK(false, false, true); else PICK(false, false, false); } }
#undef PICK
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kWarpsPerCta * 32, smem));
  if (per_sm < 1) return fail(HHG_ECUDA, "viterbi kernel does not fit on an SM");
  // persistent grid: every CTA must be resident (strip items wait on their predecessor strip)
  int grid = ctx->sm_count * per_sm;
  const int need = (items + kWarpsPerCta - 1) / kWarpsPerCta;
  if (grid > need) grid = need;
  kern<<<grid, kWarpsPerCta * 32, smem, ctx->stream>>>(P);
  ctx->launches++;
  CK(cudaGetLastError());
  return HHG_OK;
}

static int plan_run_impl(hhg_ctx* ctx, hhg_plan* pl, bool timed) {
  if (!ctx || !pl) return fail(HHG_EINVAL, "hhg_plan_run: bad argument");
  if (!pl->built) return fail(HHG_EINVAL, "hhg_plan_run: the plan's last build failed");
  if (pl->q_L != ctx->q_L || pl->q_row0 != ctx->q_row0) return fail(HHG_EINVAL, "plan was made for another query (batch) geometry");
  const hhg_db* db = pl->db;
  if (pl->db_serial != db->serial) return fail(HHG_EINVAL, "hhg_plan_run: the shard was staged anew after the plan was made");
  const bool fused = pl->nm_mode >= 0;     // null model factored in per job while the operand stream is built
  if (fused && (!db->raw || !ctx->has_q_pav)) return fail(HHG_EINVAL, "fused null model needs a raw shard and query pav");
  if (!fused && !db->prepared) return fail(HHG_EINVAL, "raw db: call hhg_db_apply_null_model for the current query first");
  if (ctx->par.use_ss && (!db->has_ss || !ctx->has_ss || !ctx->has_S33))
    return fail(HHG_EINVAL, "use_ss requested but query/db/S33 carry no ss information");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  // slot tags of earlier runs never match (20-bit epoch in the tag) ... unless the epoch has wrapped since this plan's
  // slots were last cleared: then a slot left over from exactly 2^20 runs ago would look valid, so clear them once
  // per epoch window
  ctx->epoch = (ctx->epoch + 1) & 0xFFFFFu;
  if (ctx->epoch == 0) { ctx->epoch = 1; ctx->epoch_window++; }
  if (pl->bnd_epoch_window != ctx->epoch_window) {
    if (pl->d_bnd.p) CK(cudaMemsetAsync(pl->d_bnd.p, 0, pl->d_bnd.n * sizeof(BndSlot), st));
    pl->bnd_epoch_window = ctx->epoch_window;
  }
  CK(cudaMemsetAsync(pl->d_counter.p, 0, pl->waves.size() * 4, st));
  if (pl->jc_version != db->cols_version || pl->jc_nm_mode != pl->nm_mode ||
      (fused && pl->jc_query_serial != ctx->query_serial) ||
      (pl->nm_mode == 0 && memcmp(pl->jc_pb, ctx->h_pb, sizeof pl->jc_pb) != 0)) {
    // (re)build the job-interleaved operand stream: once per plan, again after every hhg_db_apply_null_model (the
    // prepared emissions changed) and, with the fused null model, for every new query batch and, with columnscore 0,
    // for every new pb (k_backtrace divides by the current one, so the forward pass must too)
    int maxL = 0;
    for (const JobDesc& jd : pl->jobs) maxL = std::max(maxL, jd.Lmax);
    dim3 grid((unsigned)pl->njobs, (unsigned)std::min(64, (maxL + 7) / 8), 1);
    k_interleave_cols<<<grid, 256, 0, st>>>(pl->d_jobs.p, pl->d_job_target.p, fused ? db->cols_raw.p : db->cols.p,
                                            db->dcol_off.p, db->dL.p, pl->d_jcols.p, pl->nm_mode, ctx->d_q_pav.p,
                                            db->pav.p, ctx->d_pb.p);
    ctx->launches++;
    CK(cudaGetLastError());
    pl->jc_version = db->cols_version;
    pl->jc_nm_mode = pl->nm_mode;
    pl->jc_query_serial = ctx->query_serial;
    memcpy(pl->jc_pb, ctx->h_pb, sizeof pl->jc_pb);
  }
  for (size_t wi = 0; wi < pl->waves.size(); ++wi) {
    const Wave& w = pl->waves[wi];
    const int nj = w.job_end - w.job_begin;
    VitParams P{};
    P.qrec = ctx->qrec.p;
    P.jobs = pl->d_jobs.p + w.job_begin;
    P.items = pl->d_items.p + w.item_begin; P.n_items = (int)(w.item_end - w.item_begin);
    P.Lt = db->dL.p;
    P.jcols = pl->d_jcols.p;
    P.njobs = nj;
    P.job_target = pl->d_job_target.p + (size_t)w.job_begin * 32;
    P.bt = pl->d_bt.p; P.bnd = pl->d_bnd.p;
    P.tag_base = ctx->epoch << 12;
    P.counter = pl->d_counter.p + wi;
    P.strip_score = pl->d_strip_score.p;     // JobDesc::ss_off is absolute
    P.strip_ij = pl->d_strip_ij.p;
    P.celloff = pl->celloff ? pl->d_co.p : nullptr;
    P.S33 = ctx->has_S33 ? ctx->S33.p : nullptr;
    P.egq = ctx->par.egq; P.egt = ctx->par.egt; P.shift = ctx->par.shift; P.ssw = ctx->par.ssw;
    P.zero = 0u;

    const int items = P.n_items;
    int rc;
    if (timed) CK(cudaEventRecord(ctx->ev[0], st));
    if (pl->R == 8) rc = launch_viterbi<8>(ctx, P, ctx->par.local != 0, ctx->par.use_ss != 0, pl->celloff, items);
    else if (pl->R == 12) rc = launch_viterbi<12>(ctx, P, ctx->par.local != 0, ctx->par.use_ss != 0, pl->celloff, items);
    else rc = launch_viterbi<16>(ctx, P, ctx->par.local != 0, ctx->par.use_ss != 0, pl->celloff, items);
    if (rc != HHG_OK) return rc;
    if (timed) CK(cudaEventRecord(ctx->ev[1], st));
    // backtrace of this wave's requests: every request whose job lies in the wave (ReqDesc::job is absolute)
    BtParams B{};
    B.n_req = pl->n;   // filtered by job range inside: simpler to launch per wave over all requests
    B.jobs = pl->d_jobs.p; B.reqs = pl->d_reqs.p;
    B.nm_mode = pl->nm_mode; B.q_pav = ctx->d_q_pav.p; B.t_pav = db->pav.p; B.pb = ctx->d_pb.p;
    B.bt = pl->d_bt.p; B.strip_score = pl->d_strip_score.p; B.strip_ij = pl->d_strip_ij.p;
    B.hits = pl->d_hits.p; B.paths = pl->d_paths.p;
    B.job_begin = w.job_begin; B.job_end = w.job_end;
    B.qrec = ctx->qrec.p; B.cols = fused ? db->cols_raw.p : db->cols.p; B.col_off = db->dcol_off.p;
    B.lg2 = ctx->lg2.p; B.diff = ctx->diff.p; B.S33 = ctx->has_S33 ? ctx->S33.p : nullptr; B.S = pl->d_S.p;
    B.corr = ctx->par.corr; B.ssw = ctx->par.ssw; B.use_ss = ctx->par.use_ss; B.ss_score_mode = (ctx->par.ssm == 2);
    const int threads = 128;
    k_backtrace<<<(pl->n + threads - 1) / threads, threads, 0, st>>>(B);
    ctx->launches++;
    CK(cudaGetLastError());
    if (timed) {
      CK(cudaEventRecord(ctx->ev[2], st));
      CK(cudaEventSynchronize(ctx->ev[2]));
      float a = 0, b = 0;
      CK(cudaEventElapsedTime(&a, ctx->ev[0], ctx->ev[1]));
      CK(cudaEventElapsedTime(&b, ctx->ev[1], ctx->ev[2]));
      pl->ms_viterbi += a;
      pl->ms_backtrace += b;
    }
  }
  return HHG_OK;
}

int hhg_plan_run(hhg_ctx* ctx, hhg_plan* pl) { return plan_run_impl(ctx, pl, false); }

// Same as hhg_plan_run but brackets every forward-pass and backtrace launch with CUDA events on the
// context stream and returns their summed device times (ms).  Synchronises; used by bench.py for the
// per-kernel roofline figure.
int hhg_plan_run_timed(hhg_ctx* ctx, hhg_plan* pl, float* ms_viterbi, float* ms_backtrace) {
  if (!ctx || !pl) return fail(HHG_EINVAL, "hhg_plan_run_timed: bad argument");
  for (int k = 0; k < 3; ++k)
    if (!ctx->ev[k]) CK(cudaEventCreate(&ctx->ev[k]));
  pl->ms_viterbi = pl->ms_backtrace = 0;
  int rc = plan_run_impl(ctx, pl, true);
  if (rc != HHG_OK) return rc;
  if (ms_viterbi) *ms_viterbi = pl->ms_viterbi;
  if (ms_backtrace) *ms_backtrace = pl->ms_backtrace;
  return HHG_OK;
}

int hhg_plan_fetch(hhg_ctx* ctx, hhg_plan* pl, hhg_hit* hits, uint8_t* paths, size_t paths_cap) {
  if (!ctx || !pl || !hits) return fail(HHG_EINVAL, "hhg_plan_fetch: bad argument");
  static_assert(sizeof(hhg_hit) == sizeof(HitRec), "hhg_hit / HitRec layout");
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(hits, pl->d_hits.p, (size_t)pl->n * sizeof(HitRec), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (paths) {
    // compact on the device: only nsteps bytes per request cross PCIe (capacity is Lq+Lt+2 each)
    pl->h_compact_off.resize(pl->n);
    long long tot = 0;
    for (int k = 0; k < pl->n; ++k) { pl->h_compact_off[k] = tot; tot += hits[k].nsteps; }
    if (paths_cap < (size_t)tot) return fail(HHG_EINVAL, "paths buffer too small: need %lld bytes", tot);
    CK(pl->d_compact_off.ensure(pl->n));
    CK(pl->d_paths_compact.ensure((size_t)std::max<long long>(tot, 1)));
    CK(cudaMemcpyAsync(pl->d_compact_off.p, pl->h_compact_off.data(), (size_t)pl->n * 8, cudaMemcpyHostToDevice, ctx->stream));
    const int threads = 128;
    k_gather_paths<<<(pl->n + threads - 1) / threads, threads, 0, ctx->stream>>>(
        pl->n, pl->d_hits.p, pl->d_reqs.p, pl->d_compact_off.p, pl->d_paths.p, pl->d_paths_compact.p);
    ctx->launches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(paths, pl->d_paths_compact.p, (size_t)tot, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int k = 0; k < pl->n; ++k) hits[k].path_off = (int32_t)pl->h_compact_off[k];
  }
  return HHG_OK;
}

void* hhg_plan_hits_devptr(hhg_plan* plan) { return plan ? (void*)plan->d_hits.p : nullptr; }
hhg_plan* hhg_ctx_last_plan(hhg_ctx* ctx) { return ctx ? ctx->scratch_plan : nullptr; }

int hhg_plan_debug_bt(hhg_ctx* ctx, hhg_plan* pl, int k, uint8_t* bt) {
  if (!ctx || !pl || !bt || k < 0 || k >= pl->n) return fail(HHG_EINVAL, "hhg_plan_debug_bt: bad argument");
  if (!pl->built) return fail(HHG_EINVAL, "hhg_plan_debug_bt: the plan's last build failed");
  if (pl->waves.size() != 1) return fail(HHG_EINVAL, "debug_bt needs a single-wave plan");
  CK(cudaSetDevice(ctx->device));
  const ReqDesc& rq = pl->reqs[k];
  const JobDesc& jd = pl->jobs[rq.job];
  const int total = (rq.Lq + 1) * (rq.Lt + 1);
  DevBuf<uint8_t> tmp;
  CK(tmp.alloc(total));
  k_debug_bt<<<(total + 255) / 256, 256, 0, ctx->stream>>>(pl->d_bt.p, jd.bt_off, rq.lane, jd.Lmax, rq.Lq, rq.Lt,
                                                            tmp.p);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(bt, tmp.p, total, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

int hhg_viterbi_search(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* ids, hhg_hit* hits,
                       uint8_t* paths, size_t paths_cap, const int64_t* excl_off,
                       const int32_t* excl_i, const int32_t* excl_j) {
  if (!ctx) return fail(HHG_EINVAL, "ctx is NULL");
  if (!ctx->scratch_plan) ctx->scratch_plan = new hhg_plan();
  hhg_plan* pl = ctx->scratch_plan;
  static const bool timing = getenv("HHG_TIMING") != nullptr;   // developer aid: host-side phase times on stderr
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto t0 = now();
  int rc = plan_build(ctx, pl, db, n, ids);
  if (rc != HHG_OK) return rc;
  pl->nm_mode = -1;
  auto t1 = now();
  rc = set_exclusions(ctx, pl, excl_off, excl_i, excl_j);
  if (rc == HHG_OK) rc = hhg_plan_run(ctx, pl);
  if (timing) cudaStreamSynchronize(ctx->stream);
  auto t2 = now();
  if (rc == HHG_OK) rc = hhg_plan_fetch(ctx, pl, hits, paths, paths_cap);
  if (timing) {
    auto ms = [](decltype(t0) a, decltype(t0) b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    fprintf(stderr, "[hhg] viterbi_search n=%d: plan %.3f ms, run (device) %.3f ms, fetch %.3f ms\n", n, ms(t0, t1), ms(t1, t2), ms(t2, now()));
  }
  return rc;
}


// Query-batch search (SURVEY 8f-4): nq queries set by hhg_query_set_batch, request k aligns query req_query[k] with
// target ids[k]; ONE plan, one forward launch per memory wave with the work items of all queries in it.
// excl_*: the earlier alignments of each request, checked against that request's query and target lengths.
int hhg_viterbi_search_batch(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* req_query, const int32_t* ids,
                             int columnscore, const float* pb, hhg_hit* hits, uint8_t* paths, size_t paths_cap,
                             const int64_t* excl_off, const int32_t* excl_i, const int32_t* excl_j) {
  if (!ctx || !db || !req_query || !ids) return fail(HHG_EINVAL, "hhg_viterbi_search_batch: bad argument");
  if (!ctx->scratch_plan) ctx->scratch_plan = new hhg_plan();
  hhg_plan* pl = ctx->scratch_plan;
  int rc = plan_build(ctx, pl, db, n, ids, req_query);
  if (rc != HHG_OK) return rc;
  pl->nm_mode = -1;
  if (db->raw) {
    // every query needs its own null model: factor it in while the plan's operand stream is built
    if (columnscore < 0 || columnscore > 3) return fail(HHG_EINVAL, "hhg_viterbi_search_batch: columnscore %d", columnscore);
    if (!ctx->has_q_pav) return fail(HHG_EINVAL, "hhg_viterbi_search_batch: raw shard needs q_pav in hhg_query_set_batch");
    if (columnscore == 0 && !pb) return fail(HHG_EINVAL, "hhg_viterbi_search_batch: columnscore 0 needs pb");
    memset(ctx->h_pb, 0, sizeof ctx->h_pb);
    if (pb) memcpy(ctx->h_pb, pb, sizeof ctx->h_pb);
    CK(ctx->d_pb.ensure(20));
    CK(cudaMemcpyAsync(ctx->d_pb.p, ctx->h_pb, sizeof ctx->h_pb, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    pl->nm_mode = columnscore;
  }
  rc = set_exclusions(ctx, pl, excl_off, excl_i, excl_j);      // + the excluded regions of the context, if any
  if (rc == HHG_OK) rc = hhg_plan_run(ctx, pl);
  if (rc == HHG_OK) rc = hhg_plan_fetch(ctx, pl, hits, paths, paths_cap);
  return rc;
}

// ------------------------------------------------------------------------------ multi-GPU: NCCL behind the C-ABI
// NCCL is bound at run time (dlopen "libnccl.so.2"): a single-GPU user needs no NCCL at all, and inside a process
// that already loaded a copy (e.g. PyTorch's bundled one) the same copy is used.  Only the stable core entry
// points are needed; their prototypes are restated here (nccl.h: ncclGetUniqueId :146, ncclCommInitRank :160,
// ncclCommDestroy :181, ncclAllGather :425, ncclAllReduce, ncclGetErrorString).
namespace {
typedef struct ncclComm* nccl_comm_t;
typedef struct { char internal[128]; } nccl_uid_t;
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(nccl_uid_t*) = nullptr;
  int (*CommInitRank)(nccl_comm_t*, int, nccl_uid_t, int) = nullptr;
  int (*CommDestroy)(nccl_comm_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
std::once_flag g_nccl_once;
const char* g_nccl_err = nullptr;

int nccl_load() {
  std::call_once(g_nccl_once, [] {
    const char* names[] = {getenv("HHG_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) {
      if (!nm) continue;
      g_nccl.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
      if (g_nccl.lib) break;
    }
    if (!g_nccl.lib) { g_nccl_err = "libnccl.so.2 not found (set HHG_NCCL_LIB)"; return; }
#define SYM(f) *(void**)(&g_nccl.f) = dlsym(g_nccl.lib, "nccl" #f); if (!g_nccl.f) g_nccl_err = "NCCL symbol nccl" #f " missing"
    SYM(GetUniqueId); SYM(CommInitRank); SYM(CommDestroy); SYM(AllGather); SYM(AllReduce); SYM(GetErrorString);
#undef SYM
  });
  return g_nccl_err ? fail(HHG_ECUDA, "%s", g_nccl_err) : HHG_OK;
}
#define NCK(expr)                                                                                           \
  do {                                                                                                      \
    int r__ = (expr);                                                                                       \
    if (r__ != 0) return fail(HHG_ECUDA, "%s: NCCL error %d (%s)", #expr, r__, g_nccl.GetErrorString(r__)); \
  } while (0)
}  // namespace

struct hhg_comm {
  int rank = 0, world = 1, device = 0;
  nccl_comm_t comm = nullptr;
};

int hhg_comm_unique_id(void* id128) {
  if (!id128) return fail(HHG_EINVAL, "hhg_comm_unique_id: id is NULL");
  int rc = nccl_load();
  if (rc != HHG_OK) return rc;
  nccl_uid_t id;
  NCK(g_nccl.GetUniqueId(&id));
  memcpy(id128, &id, sizeof id);
  return HHG_OK;
}

int hhg_comm_create(hhg_ctx* ctx, int rank, int world, const void* id128, hhg_comm** out) {
  if (!ctx || !out || world < 1 || rank < 0 || rank >= world || (world > 1 && !id128))
    return fail(HHG_EINVAL, "hhg_comm_create: bad argument");
  std::unique_ptr<hhg_comm> c(new hhg_comm());
  c->rank = rank; c->world = world; c->device = ctx->device;
  if (world > 1) {
    int rc = nccl_load();
    if (rc != HHG_OK) return rc;
    CK(cudaSetDevice(ctx->device));
    nccl_uid_t id;
    memcpy(&id, id128, sizeof id);
    NCK(g_nccl.CommInitRank(&c->comm, world, id, rank));
  }
  *out = c.release();
  return HHG_OK;
}

int hhg_comm_destroy(hhg_comm* c) {
  if (!c) return HHG_OK;
  if (c->comm) { cudaSetDevice(c->device); g_nccl.CommDestroy(c->comm); }
  delete c;
  return HHG_OK;
}

int hhg_comm_rank(const hhg_comm* c) { return c ? c->rank : 0; }
int hhg_comm_world(const hhg_comm* c) { return c ? c->world : 1; }

// Top-K of the last run of `plan`, merged over all ranks of `comm` (NULL / world 1: this GPU only).
static int plan_topk_impl(hhg_ctx* ctx, hhg_plan* pl, hhg_comm* comm, int K, int by_hit_score, const float* user_key,
                          int32_t id_base, const int32_t* global_ids, hhg_topk_rec* out, int* n_out) {
  static_assert(sizeof(hhg_topk_rec) == sizeof(TopkRec), "hhg_topk_rec / TopkRec layout");
  if (!ctx || !pl || K < 1 || !out || !n_out) return fail(HHG_EINVAL, "hhg_plan_topk: bad argument");
  if (comm && comm->world > 1 && comm->device != ctx->device) return fail(HHG_EINVAL, "hhg_plan_topk: comm lives on another device");
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int n = pl->n;
  const int world = comm ? comm->world : 1, rank = comm ? comm->rank : 0;
  const int kl = std::min(K, n);
  CK(pl->d_keys.ensure((size_t)n)); CK(pl->d_topk_state.ensure(1));
  CK(pl->d_topk_local.ensure((size_t)K)); CK(pl->d_topk_all.ensure((size_t)K * world));
  if (global_ids) {
    CK(pl->d_gids.ensure((size_t)n));
    CK(cudaMemcpyAsync(pl->d_gids.p, global_ids, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  }
  if (user_key) {
    CK(pl->d_user_key.ensure((size_t)n));
    CK(cudaMemcpyAsync(pl->d_user_key.p, user_key, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  }
  TopkState init{};
  init.krem = (unsigned)kl;
  CK(cudaMemcpyAsync(pl->d_topk_state.p, &init, sizeof init, cudaMemcpyHostToDevice, st));
  const int threads = 256, blocks = (n + threads - 1) / threads;
  k_topk_keys<<<blocks, threads, 0, st>>>(n, pl->d_hits.p, by_hit_score, id_base, global_ids ? pl->d_gids.p : nullptr,
                                            user_key ? pl->d_user_key.p : nullptr, pl->d_keys.p);
  const int hblocks = std::min(blocks, ctx->sm_count * 4);
  for (int p = 7; p >= 0; --p) {
    k_topk_hist<<<hblocks, threads, 0, st>>>(n, pl->d_keys.p, p, pl->d_topk_state.p);
    k_topk_scan<<<1, 256, 0, st>>>(pl->d_topk_state.p);
  }
  k_topk_emit<<<blocks, threads, 0, st>>>(n, pl->d_keys.p, pl->d_hits.p, rank, pl->d_topk_state.p, pl->d_topk_local.p, K);
  ctx->launches += 18;
  if (kl < K) { k_topk_pad<<<(K - kl + 255) / 256, 256, 0, st>>>(pl->d_topk_local.p, kl, K); ctx->launches++; }
  CK(cudaGetLastError());
  const TopkRec* src = pl->d_topk_local.p;
  if (world > 1) {
    NCK(g_nccl.AllGather(pl->d_topk_local.p, pl->d_topk_all.p, (size_t)K * sizeof(TopkRec), /*ncclChar*/ 0, comm->comm, st));
    src = pl->d_topk_all.p;
  }
  std::vector<TopkRec> all((size_t)K * world);
  CK(cudaMemcpyAsync(all.data(), src, all.size() * sizeof(TopkRec), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  // merge: keys are unique and totally ordered (score descending, global id ascending)
  all.erase(std::remove_if(all.begin(), all.end(), [](const TopkRec& r) { return r.target < 0; }), all.end());
  std::sort(all.begin(), all.end(), [](const TopkRec& a, const TopkRec& b) { return a.key < b.key; });
  const int m = (int)std::min<size_t>(all.size(), (size_t)K);
  memcpy(out, all.data(), (size_t)m * sizeof(TopkRec));
  *n_out = m;
  return HHG_OK;
}

int hhg_plan_topk(hhg_ctx* ctx, hhg_plan* pl, hhg_comm* comm, int K, int by_hit_score, int32_t id_base,
                  const int32_t* global_ids, hhg_topk_rec* out, int* n_out) {
  return plan_topk_impl(ctx, pl, comm, K, by_hit_score, nullptr, id_base, global_ids, out, n_out);
}

int hhg_plan_topk_by_key(hhg_ctx* ctx, hhg_plan* pl, hhg_comm* comm, int K, const float* key, int32_t id_base,
                         const int32_t* global_ids, hhg_topk_rec* out, int* n_out) {
  if (!key) return fail(HHG_EINVAL, "hhg_plan_topk_by_key: key is NULL");
  return plan_topk_impl(ctx, pl, comm, K, 0, key, id_base, global_ids, out, n_out);
}

// State strings of the merged list: out[r*width .. ] = path of recs[r] (nsteps bytes, zero padded), on every rank.
int hhg_plan_topk_paths(hhg_ctx* ctx, hhg_plan* pl, hhg_comm* comm, int n_rec, const hhg_topk_rec* recs, int width,
                        uint8_t* out) {
  if (!ctx || !pl || n_rec < 0 || !recs || width < 1 || !out) return fail(HHG_EINVAL, "hhg_plan_topk_paths: bad argument");
  if (n_rec == 0) return HHG_OK;
  CK(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const int world = comm ? comm->world : 1, rank = comm ? comm->rank : 0;
  CK(pl->d_topk_all.ensure((size_t)n_rec));
  CK(pl->d_topk_paths.ensure((size_t)n_rec * width));
  CK(cudaMemcpyAsync(pl->d_topk_all.p, recs, (size_t)n_rec * sizeof(TopkRec), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(pl->d_topk_paths.p, 0, (size_t)n_rec * width, st));
  k_topk_paths<<<n_rec, 128, 0, st>>>(n_rec, pl->d_topk_all.p, rank, pl->d_paths.p, width, pl->d_topk_paths.p);
  ctx->launches++;
  CK(cudaGetLastError());
  if (world > 1)
    NCK(g_nccl.AllReduce(pl->d_topk_paths.p, pl->d_topk_paths.p, (size_t)n_rec * width, /*ncclUint8*/ 1, /*ncclSum*/ 0, comm->comm, st));
  CK(cudaMemcpyAsync(out, pl->d_topk_paths.p, (size_t)n_rec * width, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return HHG_OK;
}

// ------------------------------------------------------------------------------------ MAC realignment
// HMM::Log2LinTransitionProbs(1.0) (src/hhhmm.cpp:2305-2313) for host arrays: tr = pow(2.0f, 1.0f * tr), which with
// float arguments is the C library's powf.  Host only.
int hhg_log2lin(int64_t n, const float* in, float* out) {
  if (n < 0 || !in || !out) return fail(HHG_EINVAL, "hhg_log2lin: bad argument");
  for (int64_t k = 0; k < n; ++k) out[k] = ::powf(2.0f, 1.0f * in[k]);
  return HHG_OK;
}

// The queries of the following realignments: p as it is, the linear transitions with the boundary rows reset like
// PosteriorDecoderRunner::initializeQueryHMMTransitions (src/hhposteriordecoderrunner.cpp:145-155).  q_pav[nq*20]
// (HMM::pav) is needed only to realign over a raw shard.
static int mac_query_set_impl(hhg_ctx* ctx, const char* who, int nq, const int32_t* Lq, const float* const* q_p,
                              const float* const* q_tr_lin, const float* q_pav) {
  if (!ctx || nq < 1 || !Lq || !q_p || !q_tr_lin) return fail(HHG_EINVAL, "%s: bad argument", who);
  for (int q = 0; q < nq; ++q)
    if (Lq[q] < 1 || Lq[q] > 32767 || !q_p[q] || !q_tr_lin[q]) return fail(HHG_EINVAL, "%s: bad query %d", who, q);
  CK(cudaSetDevice(ctx->device));
  std::vector<long long> off(2 * (size_t)nq);
  long long np = 0, ntr = 0;
  for (int q = 0; q < nq; ++q) {
    off[q] = np; np += (long long)(Lq[q] + 2) * 20;
    off[nq + q] = ntr; ntr += (long long)(Lq[q] + 1) * 7;
  }
  std::vector<float> hp((size_t)np), htr((size_t)ntr);
  for (int q = 0; q < nq; ++q) {
    memcpy(hp.data() + off[q], q_p[q], (size_t)(Lq[q] + 2) * 80);
    float* tr = htr.data() + off[nq + q];
    memcpy(tr, q_tr_lin[q], (size_t)(Lq[q] + 1) * 28);
    // (enum order M2M,M2I,M2D,I2M,I2I,D2M,D2D)
    tr[1] = tr[2] = tr[3] = tr[4] = tr[5] = tr[6] = 0.0f;
    float* e = tr + (size_t)Lq[q] * 7;
    e[0] = 1.0f; e[1] = e[2] = e[3] = e[4] = 0.0f; e[5] = 1.0f; e[6] = 0.0f;
  }
  ctx->mac_nq = 0;                                          // no query until the upload went through
  CK(ctx->mac_qp.ensure((size_t)np)); CK(ctx->mac_qtr.ensure((size_t)ntr));
  CK(ctx->mac_qL_d.ensure((size_t)nq)); CK(ctx->mac_qoff.ensure(off.size()));
  CK(cudaMemcpyAsync(ctx->mac_qp.p, hp.data(), hp.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->mac_qtr.p, htr.data(), htr.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->mac_qL_d.p, Lq, (size_t)nq * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->mac_qoff.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  if (q_pav) {
    CK(ctx->mac_q_pav.ensure((size_t)nq * 20));
    CK(cudaMemcpyAsync(ctx->mac_q_pav.p, q_pav, (size_t)nq * 80, cudaMemcpyHostToDevice, ctx->stream));
  }
  CK(cudaStreamSynchronize(ctx->stream));
  ctx->mac_qL.assign(Lq, Lq + nq);
  ctx->mac_has_q_pav = q_pav != nullptr;
  ctx->mac_nq = nq;
  return HHG_OK;
}

int hhg_mac_query_set(hhg_ctx* ctx, int Lq, const float* q_p, const float* q_tr_lin) {
  const int32_t L1 = Lq;
  return mac_query_set_impl(ctx, "hhg_mac_query_set", 1, &L1, &q_p, &q_tr_lin, nullptr);
}

int hhg_mac_query_set_batch(hhg_ctx* ctx, int nq, const int32_t* Lq, const float* const* q_p,
                            const float* const* q_tr_lin, const float* q_pav) {
  return mac_query_set_impl(ctx, "hhg_mac_query_set_batch", nq, Lq, q_p, q_tr_lin, q_pav);
}

// The one host path of hhg_mac_realign (batch == false: every request realigns query 0 over the shard's prepared
// records) and hhg_mac_realign_batch (request r realigns query req_query[r]; over a raw shard the null model of that
// query is applied to a copy of the template's records, k_mac_gather_cols).
static int mac_realign_impl(hhg_ctx* ctx, const hhg_db* db, bool batch, int n, const int32_t* req_query,
                            const int32_t* target, const int32_t* vit, const int64_t* vit_off, const int32_t* vit_i,
                            const int32_t* vit_j, const int64_t* excl_off, const int32_t* excl_i, const int32_t* excl_j,
                            int columnscore, const float* pb, const hhg_mac_params* par, hhg_mac_hit* hits,
                            int32_t* out_i, int32_t* out_j, uint8_t* out_states, float* out_post, size_t path_cap) {
  const char* who = batch ? "hhg_mac_realign_batch" : "hhg_mac_realign";
  if (!ctx || !db || n <= 0 || (batch && !req_query) || !target || !vit || !vit_off || !vit_i || !vit_j || !par ||
      !hits || !out_i || !out_j || !out_states || !out_post)
    return fail(HHG_EINVAL, "%s: bad argument", who);
  if (ctx->mac_nq <= 0)
    return fail(HHG_EINVAL, "%s: call %s first", who, batch ? "hhg_mac_query_set_batch" : "hhg_mac_query_set");
  const bool fuse = batch && db->raw;
  if (!fuse && !db->prepared) return fail(HHG_EINVAL, "%s: shard has no null model applied", who);
  if (fuse) {
    // every query needs its own null model (columnscore / pb as in hhg_viterbi_search_batch)
    if (columnscore < 0 || columnscore > 3) return fail(HHG_EINVAL, "%s: columnscore %d", who, columnscore);
    if (!ctx->mac_has_q_pav) return fail(HHG_EINVAL, "%s: raw shard needs q_pav in hhg_mac_query_set_batch", who);
    if (columnscore == 0 && !pb) return fail(HHG_EINVAL, "%s: columnscore 0 needs pb", who);
  }
  if (excl_off && (!excl_i || !excl_j)) return fail(HHG_EINVAL, "%s: excl_off without excl_i/excl_j", who);
  CK(cudaSetDevice(ctx->device));
  const bool timing = getenv("HHG_MAC_TIMING") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto ms_since = [](std::chrono::steady_clock::time_point a) {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count();
  };
  const auto t_begin = now();
  double t_prep = 0, t_lin = 0, t_kern = 0;
  static_assert(sizeof(MacHitOut) == sizeof(hhg_mac_hit), "hhg_mac_hit layout");
  std::vector<int> Lt(n), rq(n), Lqr(n);
  for (int r = 0; r < n; ++r) {
    const int q = req_query ? req_query[r] : 0;
    if (q < 0 || q >= ctx->mac_nq) return fail(HHG_EINVAL, "%s: request %d: query index %d out of range (%d queries)", who, r, q, ctx->mac_nq);
    const int t = target[r];
    if (t < 0 || t >= db->n) return fail(HHG_EINVAL, "request %d: target id %d out of range", r, t);
    if (db->L[t] < 1) return fail(HHG_EINVAL, "request %d: slot %d of the staged shard is empty", r, t);
    const int L = db->L[t], Lq = ctx->mac_qL[q];
    const int32_t* v = vit + (size_t)r * 5;
    const long long ns = vit_off[r + 1] - vit_off[r];
    if (v[4] != ns || ns < 0) return fail(HHG_EINVAL, "request %d: nsteps %d but %lld path entries", r, v[4], ns);
    if (v[0] < 1 || v[1] > Lq || v[0] > v[1] || v[2] < 1 || v[3] > L || v[2] > v[3])
      return fail(HHG_EINVAL, "request %d: Viterbi end points (%d-%d, %d-%d) outside 1..%d x 1..%d", r, v[0], v[1], v[2], v[3], Lq, L);
    for (long long s = vit_off[r]; s < vit_off[r + 1]; ++s)
      if (vit_i[s] < 1 || vit_i[s] > Lq || vit_j[s] < 1 || vit_j[s] > L)
        return fail(HHG_EINVAL, "request %d: Viterbi path leaves the matrix 1..%d x 1..%d", r, Lq, L);
    if (excl_off)
      for (long long s = excl_off[r]; s < excl_off[r + 1]; ++s)
        if (excl_i[s] < 1 || excl_i[s] > Lq || excl_j[s] < 1 || excl_j[s] > L)
          return fail(HHG_EINVAL, "request %d: excluded alignment leaves the matrix", r);
    Lt[r] = L; rq[r] = q; Lqr[r] = Lq;
  }
  // template transitions do not depend on the query: one slot per distinct target of the call
  std::vector<int> uniq(target, target + n);
  std::sort(uniq.begin(), uniq.end());
  uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
  const int nu = (int)uniq.size();
  std::vector<long long> u_rec0(nu), u_tr_off(nu);
  std::vector<int> u_L(nu);
  long long ntr = 0;
  for (int u = 0; u < nu; ++u) {
    u_rec0[u] = db->col_off[uniq[u]]; u_L[u] = db->L[uniq[u]];
    u_tr_off[u] = ntr; ntr += (long long)(u_L[u] + 1) * 7;
  }
  // memory waves: requests in order, each wave's scratch (posterior 4 + cell-off 1 + backtrace 1 bytes per cell, the
  // global row buffers, the scale factors and, over a raw shard, the template's records) within max_bt_bytes; a request
  // larger than that runs alone.  Offsets into the scratch are relative to the request's wave.
  std::vector<long long> rec0(n), tr_off(n), cell_off(n), row_off(n), scale_off(n), path_off(n);
  std::vector<int> wave_begin;
  long long npath = 0, ncell_max = 0, nrow_max = 0, nscale_max = 0, nrec_max = 0;
  {
    long long ncell = 0, nrow = 0, nscale = 0, nrec = 0, bytes = 0;
    for (int r = 0; r < n; ++r) {
      const int L = Lt[r], Lq = Lqr[r];
      const long long cells = (long long)(Lq + 1) * (L + 1);
      const long long rows = 11LL * (L + 3) + (L + 3 + 7) / 8 + 1;   // + the cell-off row of the fallback path
      const long long b = 6 * cells + 8 * rows + 8LL * (Lq + 3) + (fuse ? 112LL * L : 0);
      if (r == 0 || (bytes > 0 && bytes + b > (long long)ctx->max_bt_bytes)) {
        wave_begin.push_back(r);
        ncell = nrow = nscale = nrec = bytes = 0;
      }
      tr_off[r] = u_tr_off[std::lower_bound(uniq.begin(), uniq.end(), target[r]) - uniq.begin()];
      rec0[r] = fuse ? nrec : db->col_off[target[r]];
      cell_off[r] = ncell; row_off[r] = nrow; scale_off[r] = nscale; path_off[r] = npath;
      ncell += cells; nrow += rows; nscale += Lq + 3; nrec += fuse ? L : 0; bytes += b;
      npath += (long long)Lq + L + 2;
      ncell_max = std::max(ncell_max, ncell); nrow_max = std::max(nrow_max, nrow);
      nscale_max = std::max(nscale_max, nscale); nrec_max = std::max(nrec_max, nrec);
    }
    wave_begin.push_back(n);
  }
  const int nwaves = (int)wave_begin.size() - 1;
  if ((size_t)npath > path_cap) return fail(HHG_EINVAL, "%s: path buffers hold %zu entries, %lld needed", who, path_cap, npath);
  const long long nvit = vit_off[n] - vit_off[0];
  const long long nex = excl_off ? excl_off[n] - excl_off[0] : 0;
  // device staging: one int64 block {rec0, tr_off, cell_off, row_off, scale_off, path_off, vit_off[n+1], excl_off[n+1],
  // u_rec0, u_tr_off}, one int32 block {Lt, req_query, target, vit[5n], u_L, vit_i, vit_j, excl_i, excl_j}
  std::vector<long long> h64;
  for (const auto* v : {&rec0, &tr_off, &cell_off, &row_off, &scale_off, &path_off}) h64.insert(h64.end(), v->begin(), v->end());
  for (int r = 0; r <= n; ++r) h64.push_back(vit_off[r] - vit_off[0]);
  for (int r = 0; r <= n; ++r) h64.push_back(excl_off ? excl_off[r] - excl_off[0] : 0);
  h64.insert(h64.end(), u_rec0.begin(), u_rec0.end());
  h64.insert(h64.end(), u_tr_off.begin(), u_tr_off.end());
  std::vector<int> h32;
  h32.insert(h32.end(), Lt.begin(), Lt.end());
  h32.insert(h32.end(), rq.begin(), rq.end());
  h32.insert(h32.end(), target, target + n);
  h32.insert(h32.end(), vit, vit + (size_t)n * 5);
  h32.insert(h32.end(), u_L.begin(), u_L.end());
  h32.insert(h32.end(), vit_i + vit_off[0], vit_i + vit_off[0] + nvit);
  h32.insert(h32.end(), vit_j + vit_off[0], vit_j + vit_off[0] + nvit);
  if (excl_off) {
    h32.insert(h32.end(), excl_i + excl_off[0], excl_i + excl_off[0] + nex);
    h32.insert(h32.end(), excl_j + excl_off[0], excl_j + excl_off[0] + nex);
  }
  // from here on the scratch of the previous call is overwritten
  ctx->mac_cell_off.clear(); ctx->mac_Lt.clear(); ctx->mac_req_Lq.clear(); ctx->mac_waves = 0;
  CK(ctx->mac_i64.ensure(h64.size())); CK(ctx->mac_i32.ensure(h32.size()));
  CK(ctx->mac_ttr.ensure((size_t)ntr)); CK(ctx->mac_post.ensure((size_t)ncell_max)); CK(ctx->mac_off.ensure((size_t)ncell_max));
  CK(ctx->mac_bt.ensure((size_t)ncell_max)); CK(ctx->mac_rows.ensure((size_t)nrow_max)); CK(ctx->mac_scale.ensure((size_t)nscale_max));
  if (fuse) CK(ctx->mac_cols.ensure((size_t)nrec_max * 7));
  CK(ctx->mac_out.ensure(n)); CK(ctx->mac_out_i.ensure((size_t)npath)); CK(ctx->mac_out_j.ensure((size_t)npath));
  CK(ctx->mac_out_states.ensure((size_t)npath)); CK(ctx->mac_out_post.ensure((size_t)npath));
  CK(ctx->mac_map.ensure((size_t)n));
  CK(cudaMemcpyAsync(ctx->mac_i64.p, h64.data(), h64.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->mac_i32.p, h32.data(), h32.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  if (fuse) {
    float h_pb[20] = {};
    if (pb) memcpy(h_pb, pb, sizeof h_pb);
    CK(ctx->mac_pb.ensure(20));
    CK(cudaMemcpyAsync(ctx->mac_pb.p, h_pb, sizeof h_pb, cudaMemcpyHostToDevice, ctx->stream));
  }
  const long long* d64 = ctx->mac_i64.p;
  const long long *d_rec0 = d64, *d_tr_off = d64 + n, *d_cell_off = d64 + 2 * n, *d_row_off = d64 + 3 * n,
                  *d_scale_off = d64 + 4 * n, *d_path_off = d64 + 5 * n, *d_vit_off = d64 + 6 * n,
                  *d_excl_off = d64 + 7 * n + 1, *d_u_rec0 = d64 + 8 * n + 2, *d_u_tr_off = d_u_rec0 + nu;
  const int* d32 = ctx->mac_i32.p;
  const int *d_Lt = d32, *d_req_q = d32 + n, *d_target = d32 + 2 * n, *d_vit = d32 + 3 * n, *d_u_L = d32 + 8 * n,
            *d_vit_i = d_u_L + nu, *d_vit_j = d_vit_i + nvit, *d_excl_i = d_vit_j + nvit, *d_excl_j = d_excl_i + nex;
  MacArgs base{};
  base.local = par->local ? 1 : 0; base.mact = par->mact;
  { const char* e = getenv("HHG_MAC_BANDSCAN"); base.band_scan = (e && atoi(e) == 0) ? 0 : 1; }   // default on (2.5x); 0 = full-row scans
  base.Cshift = ::pow(2.0, par->shift);                    // src/hhforwardalgorithm.cpp:16
  base.Lq = ctx->mac_qL[0]; base.q_p = ctx->mac_qp.p; base.q_tr = ctx->mac_qtr.p;
  base.q_L = ctx->mac_qL_d.p; base.q_p_off = ctx->mac_qoff.p; base.q_tr_off = ctx->mac_qoff.p + ctx->mac_nq;
  base.cols = reinterpret_cast<const ColRec*>(fuse ? ctx->mac_cols.p : db->cols.p);
  base.t_tr = ctx->mac_ttr.p;
  base.vit_i = d_vit_i; base.vit_j = d_vit_j; base.excl_i = d_excl_i; base.excl_j = d_excl_j;
  base.post = ctx->mac_post.p; base.off = ctx->mac_off.p; base.bt = ctx->mac_bt.p; base.rows = ctx->mac_rows.p;
  base.scale = ctx->mac_scale.p;
  base.out_i = ctx->mac_out_i.p; base.out_j = ctx->mac_out_j.p; base.out_states = ctx->mac_out_states.p;
  base.out_post = ctx->mac_out_post.p;
  t_prep = ms_since(t_begin);
  const auto t_lin0 = now();
  // template transitions in linear space: gather the log2 rows on the device, powf on the host (a few threads),
  // boundary rows as initializeForAlignment sets them, back to the device
  const ColRec* tr_src = reinterpret_cast<const ColRec*>(db->raw ? db->cols_raw.p : db->cols.p);
  for (int u0 = 0; u0 < nu; u0 += 65535) {
    const int m = std::min(nu - u0, 65535);
    k_mac_gather_tr<<<dim3(8, m), 128, 0, ctx->stream>>>(m, tr_src, d_u_rec0 + u0, d_u_L + u0, d_u_tr_off + u0,
                                                         ctx->mac_ttr.p);
    ctx->launches++;
  }
  {
    std::vector<float> htr((size_t)ntr);
    CK(cudaMemcpyAsync(htr.data(), ctx->mac_ttr.p, (size_t)ntr * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    host_for(nu, [&](int u) {
      float* tr = htr.data() + u_tr_off[u];
      const int L = u_L[u];
      for (int i = 1; i < L; ++i)
        for (int k = 0; k < 7; ++k) tr[(size_t)i * 7 + k] = ::powf(2.0f, 1.0f * tr[(size_t)i * 7 + k]);
      float* b = tr;                 // t.tr[0]: M2M = 1, everything else 0
      b[0] = 1.0f; b[1] = b[2] = b[3] = b[4] = b[5] = b[6] = 0.0f;
      float* e = tr + (size_t)L * 7; // t.tr[L]: M2M = D2M = 1
      e[0] = 1.0f; e[1] = e[2] = e[3] = e[4] = 0.0f; e[5] = 1.0f; e[6] = 0.0f;
      return std::string();
    });
    CK(cudaMemcpyAsync(ctx->mac_ttr.p, htr.data(), (size_t)ntr * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  t_lin = ms_since(t_lin0);
  const auto t_k0 = now();
  // -excl / -template_excl of the context apply to the realignment like they do to the Viterbi stage
  if (!ctx->ex.empty()) {
    const int rc = upload_regions(ctx);
    if (rc != HHG_OK) return rc;
    base.reg = ctx->d_ex.p; base.reg_nq = ctx->ex_nq; base.reg_nt = ctx->ex_nt;
  }
  // working set in shared memory (117 bytes per template column).  Requests whose templates fit 64 KB (Lt <= ~555)
  // run 3 warps per SM on the main stream; longer ones get their own launch with a window of up to 200 KB on an
  // auxiliary stream so that they overlap the rest; beyond that the kernel falls back to the global scratch.
  const size_t kSmall = 64 * 1024, kLarge = 200 * 1024;
  CK(cudaFuncSetAttribute(k_mac_realign, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLarge));
  if (timing) CK(ctx->mac_dbg.ensure((size_t)n * 12));
  for (int w = 0; w < nwaves; ++w) {
    const int w0 = wave_begin[w], m = wave_begin[w + 1] - w0;
    MacArgs A = base;
    A.n = m;
    A.rec0 = d_rec0 + w0; A.tr_off = d_tr_off + w0; A.cell_off = d_cell_off + w0; A.row_off = d_row_off + w0;
    A.scale_off = d_scale_off + w0; A.path_off = const_cast<long long*>(d_path_off + w0);
    A.vit_off = d_vit_off + w0; A.excl_off = excl_off ? d_excl_off + w0 : nullptr;
    A.Lt = d_Lt + w0; A.vit = d_vit + 5 * (size_t)w0; A.req_q = d_req_q + w0;
    A.out = ctx->mac_out.p + w0;
    if (timing) A.dbg = ctx->mac_dbg.p + (size_t)w0 * 12;
    const int last = w0 + m - 1;
    const long long ncell = cell_off[last] + (long long)(Lqr[last] + 1) * (Lt[last] + 1);
    CK(cudaMemsetAsync(ctx->mac_bt.p, 0, (size_t)ncell, ctx->stream));
    if (fuse) {
      for (int r0 = 0; r0 < m; r0 += 65535) {
        const int k = std::min(m - r0, 65535);
        k_mac_gather_cols<<<dim3(4, k), 128, 0, ctx->stream>>>(
            k, d_req_q + w0 + r0, d_target + w0 + r0, d_Lt + w0 + r0, db->dcol_off.p, d_rec0 + w0 + r0, db->cols_raw.p,
            db->pav.p, ctx->mac_q_pav.p, ctx->mac_pb.p, columnscore, ctx->mac_cols.p);
        ctx->launches++;
      }
    }
    k_mac_band<<<m, 256, 0, ctx->stream>>>(A);
    ctx->launches++;
    std::vector<int> small_ids, large_ids;
    size_t small_need = 0, large_need = 0;
    for (int r = 0; r < m; ++r) {
      const size_t need = (size_t)117 * (Lt[w0 + r] + 3);
      if (need <= kSmall) { small_ids.push_back(r); small_need = std::max(small_need, need); }
      else { large_ids.push_back(r); large_need = std::max(large_need, need); }
    }
    if (large_ids.empty()) {
      A.smem_rows = (int)small_need;
      k_mac_realign<<<m, 32, small_need, ctx->stream>>>(A);
      ctx->launches++;
    } else {
      std::vector<int> map(small_ids);
      map.insert(map.end(), large_ids.begin(), large_ids.end());
      int* d_map = ctx->mac_map.p + w0;
      CK(cudaMemcpyAsync(d_map, map.data(), map.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
      int arc = ctx_aux_stream(ctx);
      if (arc != HHG_OK) return arc;
      CK(cudaEventRecord(ctx->aux_ev[0], ctx->stream));              // band + inputs ready
      CK(cudaStreamWaitEvent(ctx->aux_stream, ctx->aux_ev[0], 0));
      MacArgs AL = A;
      const size_t lsm = std::min(large_need, kLarge);
      AL.smem_rows = (int)lsm;
      AL.req_map = d_map + small_ids.size();
      k_mac_realign<<<(unsigned)large_ids.size(), 32, lsm, ctx->aux_stream>>>(AL);
      CK(cudaEventRecord(ctx->aux_ev[1], ctx->aux_stream));
      if (!small_ids.empty()) {
        A.smem_rows = (int)small_need;
        A.req_map = d_map;
        k_mac_realign<<<(unsigned)small_ids.size(), 32, small_need, ctx->stream>>>(A);
      }
      CK(cudaStreamWaitEvent(ctx->stream, ctx->aux_ev[1], 0));     // the next wave reuses the scratch
      ctx->launches += small_ids.empty() ? 1 : 2;
    }
    CK(cudaGetLastError());
  }
  if (timing) { CK(cudaStreamSynchronize(ctx->stream)); t_kern = ms_since(t_k0); }
  const auto t_d0 = now();
  CK(cudaMemcpyAsync(hits, ctx->mac_out.p, (size_t)n * sizeof(MacHitOut), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(out_i, ctx->mac_out_i.p, (size_t)npath * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(out_j, ctx->mac_out_j.p, (size_t)npath * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(out_states, ctx->mac_out_states.p, (size_t)npath, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(out_post, ctx->mac_out_post.p, (size_t)npath * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (timing) {
    std::vector<long long> d((size_t)n * 12);
    CK(cudaMemcpy(d.data(), ctx->mac_dbg.p, d.size() * 8, cudaMemcpyDeviceToHost));
    int big = 0;
    for (int r = 1; r < n; ++r) if (Lt[r] > Lt[big]) big = r;
    for (int r : {0, big}) {
      fprintf(stderr, "  request %d (Lt=%d) Mcycles: fwdA %.2f fwdScan %.2f fwdEnd %.2f Pf %.2f bwdA %.2f bwdB %.2f bwdC %.2f macA %.2f macScan %.2f bt %.2f\n",
              r, Lt[r], d[r * 12 + 0] / 1e6, d[r * 12 + 1] / 1e6, d[r * 12 + 2] / 1e6, d[r * 12 + 3] / 1e6, d[r * 12 + 4] / 1e6,
              d[r * 12 + 5] / 1e6, d[r * 12 + 6] / 1e6, d[r * 12 + 7] / 1e6, d[r * 12 + 8] / 1e6, d[r * 12 + 9] / 1e6);
    }
    fprintf(stderr, "%s: n=%d waves=%d cells<=%lld per wave  prep+H2D %.2f ms, transitions (gather, powf, H2D) %.2f ms, "
            "kernels %.2f ms, D2H %.2f ms, total %.2f ms\n", who, n, nwaves, ncell_max, t_prep, t_lin, t_kern,
            ms_since(t_d0), ms_since(t_begin));
  }
  ctx->mac_cell_off = cell_off;
  ctx->mac_Lt = Lt;
  ctx->mac_req_Lq = Lqr;
  ctx->mac_waves = nwaves;
  return HHG_OK;
}

int hhg_mac_realign(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* target, const int32_t* vit,
                    const int64_t* vit_off, const int32_t* vit_i, const int32_t* vit_j, const int64_t* excl_off,
                    const int32_t* excl_i, const int32_t* excl_j, const hhg_mac_params* par, hhg_mac_hit* hits,
                    int32_t* out_i, int32_t* out_j, uint8_t* out_states, float* out_post, size_t path_cap) {
  return mac_realign_impl(ctx, db, false, n, nullptr, target, vit, vit_off, vit_i, vit_j, excl_off, excl_i, excl_j, 1,
                          nullptr, par, hits, out_i, out_j, out_states, out_post, path_cap);
}

int hhg_mac_realign_batch(hhg_ctx* ctx, const hhg_db* db, int n, const int32_t* req_query, const int32_t* target,
                          const int32_t* vit, const int64_t* vit_off, const int32_t* vit_i, const int32_t* vit_j,
                          const int64_t* excl_off, const int32_t* excl_i, const int32_t* excl_j, int columnscore,
                          const float* pb, const hhg_mac_params* par, hhg_mac_hit* hits, int32_t* out_i,
                          int32_t* out_j, uint8_t* out_states, float* out_post, size_t path_cap) {
  return mac_realign_impl(ctx, db, true, n, req_query, target, vit, vit_off, vit_i, vit_j, excl_off, excl_i, excl_j,
                          columnscore, pb, par, hits, out_i, out_j, out_states, out_post, path_cap);
}

int hhg_mac_debug_posterior(hhg_ctx* ctx, int request, float* out) {
  if (!ctx || !out || request < 0 || request >= (int)ctx->mac_cell_off.size())
    return fail(HHG_EINVAL, "hhg_mac_debug_posterior: bad argument");
  if (ctx->mac_waves > 1)
    return fail(HHG_EINVAL, "hhg_mac_debug_posterior: the last realignment ran in %d memory waves; posteriors are kept "
                "only after a single-wave call", ctx->mac_waves);
  CK(cudaSetDevice(ctx->device));
  const size_t cells = (size_t)(ctx->mac_req_Lq[request] + 1) * (ctx->mac_Lt[request] + 1);
  CK(cudaMemcpyAsync(out, ctx->mac_post.p + ctx->mac_cell_off[request], cells * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

// ------------------------------------------------------------------------------------ prefilter
int hhg_csdb_create(hhg_ctx* ctx, int n, const int32_t* L, const int64_t* off, const uint8_t* seq,
                    hhg_csdb** out) {
  if (!ctx || !out || n <= 0 || !L || !off || !seq) return fail(HHG_EINVAL, "hhg_csdb_create: bad argument");
  CK(cudaSetDevice(ctx->device));
  std::unique_ptr<hhg_csdb> holder(new hhg_csdb());
  hhg_csdb* db = holder.get();
  db->n = n;
  db->device = ctx->device;
  long long tot = 0;
  for (int k = 0; k < n; ++k) tot = std::max<long long>(tot, off[k] + L[k]);
  db->total = tot;
  CK(db->dL.alloc(n));
  CK(db->doff.alloc(n));
  CK(db->seq.alloc((size_t)tot));
  CK(db->scores.alloc(n));
  CK(cudaMemcpyAsync(db->dL.p, L, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(db->doff.p, off, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(db->seq.p, seq, (size_t)tot, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  *out = holder.release();
  return HHG_OK;
}

int hhg_csdb_destroy(hhg_csdb* db) {
  if (db) { cudaSetDevice(db->device); delete db; }
  return HHG_OK;
}

template <int WB>
static int launch_prefilter(hhg_ctx* ctx, const PfParams& P) {
  const size_t smem = (size_t)220 * WB * 32 * 4;
  auto kern = k_prefilter_ungapped<WB>;
  CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 512, smem));
  if (per_sm < 1) return fail(HHG_ECUDA, "prefilter kernel does not fit on an SM");
  kern<<<ctx->sm_count * per_sm, 512, smem, ctx->stream>>>(P);
  ctx->launches++;
  CK(cudaGetLastError());
  return HHG_OK;
}

// registers per lane of one query tile (64 positions per register): the smallest size that covers the query in one
// tile, else full 512-position tiles (225 KB of shared memory)
static int prefilter_wb(int Lq) {
  static const int kWB[] = {1, 2, 3, 4, 5, 6, 7, 8};
  for (int wb : kWB) if (Lq <= 64 * wb) return wb;
  return 8;
}

int hhg_prefilter_ungapped_run(hhg_ctx* ctx, const hhg_csdb* db, int Lq, const uint8_t* prof_host,
                               int offset, int upload_profile) {
  if (!ctx || !db || Lq < 1 || offset < 0 || offset > 255) return fail(HHG_EINVAL, "hhg_prefilter_ungapped_run: bad argument");
  const int WB = prefilter_wb(Lq);
  const int tile_pos = 64 * WB;
  const int ntiles = (Lq + tile_pos - 1) / tile_pos;
  const size_t tile_words = (size_t)220 * WB * 32;
  CK(cudaSetDevice(ctx->device));
  if (upload_profile) {
    if (!prof_host) return fail(HHG_EINVAL, "profile is NULL");
    // repack [220][Lq] bytes into [tile][220][WB][32 lanes] words: lane l of a tile owns its positions
    // l*2WB .. +2WB-1; word w = (position l*2WB+w | position l*2WB+WB+w), each as the s16 value p - offset
    std::vector<uint32_t> packed(tile_words * ntiles);
    const uint32_t pad = (uint32_t)(uint16_t)(int16_t)(-offset);
    for (int t = 0; t < ntiles; ++t)
      for (int k = 0; k < 220; ++k)
        for (int w = 0; w < WB; ++w)
          for (int l = 0; l < 32; ++l) {
            const int plo = t * tile_pos + l * 2 * WB + w, phi = plo + WB;
            const uint32_t lo = plo < Lq ? (uint32_t)(uint16_t)(int16_t)((int)prof_host[(size_t)k * Lq + plo] - offset) : pad;
            const uint32_t hi = phi < Lq ? (uint32_t)(uint16_t)(int16_t)((int)prof_host[(size_t)k * Lq + phi] - offset) : pad;
            packed[(size_t)t * tile_words + ((size_t)k * WB + w) * 32 + l] = lo | (hi << 16);
          }
    CK(ctx->pf_prof.ensure(packed.size() * 4));
    CK(cudaMemcpyAsync(ctx->pf_prof.p, packed.data(), packed.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  CK(ctx->pf_counter.ensure((size_t)ntiles));
  CK(cudaMemsetAsync(ctx->pf_counter.p, 0, 4 * (size_t)ntiles, ctx->stream));
  if (ntiles > 1) { CK(ctx->pf_edge[0].ensure((size_t)db->total)); CK(ctx->pf_edge[1].ensure((size_t)db->total)); }
  for (int t = 0; t < ntiles; ++t) {
    PfParams P{};
    P.n = db->n; P.L = db->dL.p; P.off = db->doff.p; P.seq = db->seq.p;
    P.prof32 = reinterpret_cast<const uint32_t*>(ctx->pf_prof.p) + (size_t)t * tile_words;
    P.offset = offset; P.tile = t; P.last_tile = (t == ntiles - 1);
    P.edge_in = ntiles > 1 ? ctx->pf_edge[(t + 1) & 1].p : nullptr;
    P.edge_out = ntiles > 1 ? ctx->pf_edge[t & 1].p : nullptr;
    P.scores = db->scores.p; P.counter = ctx->pf_counter.p + t;
    int rc;
    switch (WB) {
      case 1: rc = launch_prefilter<1>(ctx, P); break;
      case 2: rc = launch_prefilter<2>(ctx, P); break;
      case 3: rc = launch_prefilter<3>(ctx, P); break;
      case 4: rc = launch_prefilter<4>(ctx, P); break;
      case 5: rc = launch_prefilter<5>(ctx, P); break;
      case 6: rc = launch_prefilter<6>(ctx, P); break;
      case 7: rc = launch_prefilter<7>(ctx, P); break;
      default: rc = launch_prefilter<8>(ctx, P); break;
    }
    if (rc != HHG_OK) return rc;
  }
  return HHG_OK;
}

// Prefilter::Prefilter + init_prefilter (src/hhprefilter.cpp:28-47,314-335), the two set-up steps of the prefilter:
// (1) the column-state library: parse the text of cs219.lib (cs::ContextLibrary / ContextProfile::Read,
//     src/cs/context_profile-inl.h:81-141) and put it in linear space (cs::TransformToLin; the shipped file has
//     ISLOG F, i.e. probs = pow(2, -value/1000) in double, already linear) -> lib[k*20+a], a in the library's own
//     alphabet order A R N D C Q E G H I L K M F P S T W Y V (= the internal amino-acid order of HH-suite);
// (2) the sequences: one per ffindex entry of <db>_cs219, length = entry length - 1 (the NUL terminator).
int hhg_cs219_parse(const char* text, int64_t len, float* lib, int n_cap, int* n_states) {
  if (!text || len <= 0 || !lib || !n_states) return fail(HHG_EINVAL, "hhg_cs219_parse: bad argument");
  const char* p = text;
  const char* end = text + len;
  auto next_line = [&](const char*& b, const char*& e) {
    if (p >= end) return false;
    b = p;
    while (p < end && *p != '\n') ++p;
    e = p;
    if (p < end) ++p;
    return true;
  };
  int k = 0;
  bool is_log = false;
  const char *b, *e;
  while (next_line(b, e)) {
    if (e - b >= 5 && !strncmp(b, "ISLOG", 5)) { const char* q = b + 5; while (q < e && (*q == ' ' || *q == '\t')) ++q; is_log = (q < e && *q == 'T'); }
    if (e - b >= 5 && !strncmp(b, "PROBS", 5)) {
      if (!next_line(b, e)) break;                       // the row of the central (only) column: index + 20 values
      if (k >= n_cap) return fail(HHG_EINVAL, "hhg_cs219_parse: more than %d states", n_cap);
      const char* q = b;
      while (q < e && (*q == ' ' || *q == '\t')) ++q;
      while (q < e && *q >= '0' && *q <= '9') ++q;         // column index
      for (int a = 0; a < 20; ++a) {
        while (q < e && (*q == ' ' || *q == '\t')) ++q;
        if (q >= e) return fail(HHG_EINVAL, "hhg_cs219_parse: state %d has fewer than 20 values", k);
        double prob;
        if (*q == '*') { prob = 0.0; ++q; }
        else {
          long v = 0; bool neg = false;
          if (*q == '-') { neg = true; ++q; }
          if (q >= e || *q < '0' || *q > '9') return fail(HHG_EINVAL, "hhg_cs219_parse: state %d: not a number", k);
          while (q < e && *q >= '0' && *q <= '9') v = v * 10 + (*q++ - '0');
          if (neg) v = -v;
          prob = pow(2, static_cast<double>(-v) / 1000.0);      // ContextProfile::Read, kScale = 1000
          if (is_log) prob = exp(log(prob));                       // read as log, then TransformToLin
        }
        lib[(size_t)k * 20 + a] = (float)prob;
      }
      ++k;
    }
  }
  if (k == 0) return fail(HHG_EINVAL, "hhg_cs219_parse: no ContextProfile found");
  *n_states = k;
  return HHG_OK;
}

int hhg_csdb_create_ffindex(hhg_ctx* ctx, int n, const char* data, const int64_t* off, const int64_t* len, hhg_csdb** out) {
  if (!ctx || n <= 0 || !data || !off || !len || !out) return fail(HHG_EINVAL, "hhg_csdb_create_ffindex: bad argument");
  std::vector<int32_t> L(n);
  std::vector<int64_t> o(n);
  std::vector<uint8_t> seq;
  size_t tot = 0;
  for (int k = 0; k < n; ++k) {
    if (len[k] < 1 || off[k] < 0) return fail(HHG_EINVAL, "hhg_csdb_create_ffindex: entry %d has length %lld", k, (long long)len[k]);
    tot += (size_t)len[k] - 1;
  }
  seq.reserve(tot);
  for (int k = 0; k < n; ++k) {
    L[k] = (int32_t)(len[k] - 1);                        // length[n] = entry->length - 1, :328
    o[k] = (int64_t)seq.size();
    seq.insert(seq.end(), (const uint8_t*)data + off[k], (const uint8_t*)data + off[k] + L[k]);
  }
  return hhg_csdb_create(ctx, n, L.data(), o.data(), seq.data(), out);
}

// Host-side query profile of the prefilter (once per query; Prefilter::stripe_query_profile,
// src/hhprefilter.cpp:356-424) in the LINEAR layout prof[k*Lq+pos]: 219 column states + the ANY state.
// q_p is HMM::p of the (prefilter-pseudocount) query, i.e. float[(Lq+2)*20]; note the reference indexes
// the 1-based p array with a 0-based position (SURVEY App. D-4), reproduced here.  lib219: the 219x20
// linear column-state probabilities of cs219.lib (cs::TransformToLin).
static inline float flog2_host(float x) {       // flog2, src/util-inl.h:83-93 (double polynomial constants)
  if (x <= 0) return -128;
  uint32_t u; memcpy(&u, &x, 4);
  float e = (float)((int)((u & 0x7F800000u) >> 23) - 0x7f);
  u = (u & 0x007FFFFFu) | 0x3f800000u; memcpy(&x, &u, 4);
  x -= 1.0;
  x *= (1.441740 + x * (-0.7077702 + x * (0.4123442 + x * (-0.1903190 + x * 0.0440047))));
  return x + e;
}

int hhg_prefilter_build_profile(int Lq, const float* q_p, const float* q_pav, const float* lib219,
                                int score_offset, int bit_factor, uint8_t* prof) {
  if (Lq < 1 || !q_p || !q_pav || !lib219 || !prof) return fail(HHG_EINVAL, "hhg_prefilter_build_profile: bad argument");
  for (int k = 0; k < 219; ++k)
    for (int pos = 0; pos < Lq; ++pos) {
      float sum = 0;
      for (int a = 0; a < 20; ++a) sum += ((q_p[(size_t)pos * 20 + a] * lib219[k * 20 + a]) / q_pav[a]);
      float dummy = flog2_host(sum) * bit_factor + score_offset + 0.5;
      prof[(size_t)k * Lq + pos] = dummy > 255.0 ? 255 : (dummy < 0 ? 0 : (uint8_t)dummy);
    }
  for (int pos = 0; pos < Lq; ++pos) prof[(size_t)219 * Lq + pos] = (uint8_t)(score_offset - 1);
  return HHG_OK;
}

// Stage-1 length correction of Prefilter::prefilter_db (src/hhprefilter.cpp:477).
int hhg_prefilter_corrected_score(int raw, int Lq, int Lt, int bit_factor) {
  return raw - (int)(bit_factor * (flog2_host((float)Lq) + flog2_host((float)Lt)));
}

// Stage-2 E-value of Prefilter::prefilter_db (src/hhprefilter.cpp:529):
//   evalue = (double)num_dbs * LQ * length * fpow2(-score / bit_factor)   with INTEGER division (App. D-6)
// fpow2: src/util-inl.h:190-214.
static inline float fpow2_host(float x) {
  if (x >= FLT_MAX_EXP) return FLT_MAX;
  if (x <= FLT_MIN_EXP) return 0.0f;
  float tx = (x - 0.5f) + (3 << 22);
  uint32_t ut; memcpy(&ut, &tx, 4);
  int lx = (int)(ut - 0x4b400000u);
  float dx = x - (float)lx;
  x = 1.0f + dx * (0.693019f + dx * (0.241404f + dx * (0.0520749f + dx * 0.0134929f)));
  uint32_t ux; memcpy(&ux, &x, 4);
  ux += ((uint32_t)lx << 23);
  memcpy(&x, &ux, 4);
  return x;
}

double hhg_prefilter_evalue(int score, long long num_dbs, int Lq, int Lt, int bit_factor) {
  const double factor = (double)num_dbs * Lq;
  return factor * Lt * fpow2_host(-score / bit_factor);
}

// Batch forms of the two host-side formulas (1M-sequence shards: no per-element FFI calls).
int hhg_prefilter_corrected_scores(int n, const int32_t* raw, const int32_t* L, int Lq, int bit_factor,
                                   int32_t* out) {
  if (n < 0 || !raw || !L || !out) return fail(HHG_EINVAL, "hhg_prefilter_corrected_scores: bad argument");
  const float lq = flog2_host((float)Lq);
  for (int k = 0; k < n; ++k) out[k] = raw[k] - (int)(bit_factor * (lq + flog2_host((float)L[k])));
  return HHG_OK;
}

int hhg_prefilter_evalues(int n, const int32_t* score, const int32_t* L, long long num_dbs, int Lq,
                          int bit_factor, double* out) {
  if (n < 0 || !score || !L || !out) return fail(HHG_EINVAL, "hhg_prefilter_evalues: bad argument");
  for (int k = 0; k < n; ++k) out[k] = hhg_prefilter_evalue(score[k], num_dbs, Lq, L[k], bit_factor);
  return HHG_OK;
}

// Gapped stage 2 on the GPU for `n` selected sequences (ids == NULL: the first n of the shard).
// gap_open is the reference's gapOpen argument = prefilter_gap_open + prefilter_gap_extend (:456).
int hhg_prefilter_sw(hhg_ctx* ctx, const hhg_csdb* db, int n, const int32_t* ids, int Lq,
                     const uint8_t* prof, int gap_open, int gap_extend, int bias, int32_t* scores) {
  if (!ctx || !db || n < 1 || Lq < 1 || !prof || !scores) return fail(HHG_EINVAL, "hhg_prefilter_sw: bad argument");
  const int W = (Lq + 31) / 32;
  const size_t prof_bytes = (size_t)220 * W * 32;
  const size_t work_bytes = (size_t)8 * 3 * W * 32;             // H/H/E columns of the 8 warps of a CTA
  const bool prof_smem = prof_bytes + work_bytes <= 227 * 1024;   // else the striped profile is read through L1/L2
  const size_t smem = (prof_smem ? prof_bytes : 0) + work_bytes;
  if (smem > 227 * 1024) return fail(HHG_EINVAL, "prefilter sw: query length %d too long (working columns exceed shared memory)", Lq);
  CK(cudaSetDevice(ctx->device));
  for (int k = 0; ids && k < n; ++k)
    if (ids[k] < 0 || ids[k] >= db->n) return fail(HHG_EINVAL, "prefilter sw: id %d out of range", ids[k]);
  std::vector<uint8_t> striped(prof_bytes);
  for (int k = 0; k < 220; ++k)
    for (int j = 0; j < W; ++j)
      for (int l = 0; l < 32; ++l) {
        const int pos = l * W + j;
        striped[((size_t)k * W + j) * 32 + l] = pos < Lq ? prof[(size_t)k * Lq + pos] : (uint8_t)bias;
      }
  CK(ctx->sw_prof.ensure(prof_bytes)); CK(ctx->sw_scores.ensure(n)); CK(ctx->pf_counter.ensure(1));
  if (ids) CK(ctx->sw_ids.ensure(n));
  CK(cudaMemcpyAsync(ctx->sw_prof.p, striped.data(), prof_bytes, cudaMemcpyHostToDevice, ctx->stream));
  if (ids) CK(cudaMemcpyAsync(ctx->sw_ids.p, ids, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->pf_counter.p, 0, 4, ctx->stream));
  SwParams P{};
  P.n = n; P.ids = ids ? ctx->sw_ids.p : nullptr; P.L = db->dL.p; P.off = db->doff.p; P.seq = db->seq.p;
  P.prof = ctx->sw_prof.p; P.W = W; P.gap_open = gap_open; P.gap_extend = gap_extend; P.bias = bias;
  P.scores = ctx->sw_scores.p; P.counter = ctx->pf_counter.p;
  void (*swk)(const SwParams) = prof_smem ? k_prefilter_sw<true> : k_prefilter_sw<false>;
  CK(cudaFuncSetAttribute(swk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, swk, 256, smem));
  if (per_sm < 1) return fail(HHG_ECUDA, "prefilter sw kernel does not fit on an SM");
  const int grid = std::min(ctx->sm_count * per_sm, (n + 7) / 8);
  swk<<<grid, 256, smem, ctx->stream>>>(P);
  ctx->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(scores, ctx->sw_scores.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));   // `striped` is a host temporary
  return HHG_OK;
}

// Stage 1 of Prefilter::prefilter_db selected on the device (src/hhprefilter.cpp:477-506) for nq rows of raw ungapped
// scores (raw: [nq][db->n] on the device).  One launch corrects and histograms every row; the host reads each row's cut
// off its histogram, which also gives the exact sizes of the row's lists A (above the cut) and B (at the cut); one
// launch compacts the survivors of every row into its own region, and only they travel to the host, where each row is
// put in the reference's order (descending by (score, index): comparePair + reverse, :489-490; ties at the cut: larger
// index first).  off[nq+1]: first output slot of each row, filled before the capacity check.
static int select_rows(hhg_ctx* ctx, const hhg_csdb* db, int nq, const int32_t* Lq, const int* raw, int bit_factor,
                       int smax_thresh, int min_hits, int32_t* ids, int32_t* scores, int cap, int32_t* off,
                       const char* who) {
  auto bin_of = [](long long score) { return (int)std::min<long long>(std::max<long long>(score + kPfHistBias, 0), kPfHistBins - 1); };
  if (bin_of(smax_thresh) <= 0 || bin_of(smax_thresh) >= kPfHistBins - 1)
    return fail(HHG_EINVAL, "%s: smax_thresh %d outside the histogram range", who, smax_thresh);
  CK(cudaSetDevice(ctx->device));
  const int n = db->n;
  CK(ctx->pf_corr.ensure((size_t)nq * n));
  CK(ctx->pf_hist.ensure((size_t)nq * (kPfHistBins + 2)));
  CK(ctx->pfb_flog2.ensure(nq));
  unsigned* counters = ctx->pf_hist.p + (size_t)nq * kPfHistBins;   // [nq][2]: list A / list B
  std::vector<float> lq(nq);
  for (int q = 0; q < nq; ++q) lq[q] = flog2_host((float)Lq[q]);
  CK(cudaMemcpyAsync(ctx->pfb_flog2.p, lq.data(), (size_t)nq * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->pf_hist.p, 0, (size_t)nq * (kPfHistBins + 2) * 4, ctx->stream));
  const int bx = std::min((n + 255) / 256, std::max(1, ctx->sm_count * 8 / nq));
  k_pf_correct_hist<<<dim3(bx, nq), 256, 0, ctx->stream>>>(n, db->dL.p, raw, ctx->pfb_flog2.p, bit_factor,
                                                            ctx->pf_corr.p, ctx->pf_hist.p);
  ctx->launches++;
  CK(cudaGetLastError());
  std::vector<unsigned> hist((size_t)nq * kPfHistBins);
  CK(cudaMemcpyAsync(hist.data(), ctx->pf_hist.p, hist.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  // keep while count < min_hits or score > smax_thresh  ==  everything above the threshold, but at least the
  // min_hits best: cut = min(smax_thresh, score of the min_hits-th best); ties at the cut resolved by index
  std::vector<PfCut> cuts(nq);
  std::vector<long long> n_a(nq), n_b(nq), want_eq(nq);
  long long tot_a = 0, tot_b = 0, total = 0;
  const long long need = std::min<long long>(min_hits, n);
  for (int q = 0; q < nq; ++q) {
    const unsigned* h = hist.data() + (size_t)q * kPfHistBins;
    long long above = 0;
    for (int b = bin_of(smax_thresh) + 1; b < kPfHistBins; ++b) above += h[b];
    int cut = smax_thresh, take_eq = 0;
    if (above < need) {
      above = 0;
      int b = kPfHistBins - 1;
      for (; b >= 0; --b) {                         // highest score whose class completes the first `need` entries
        if (above + h[b] >= need) break;
        above += h[b];
      }
      if (b <= 0 || b >= kPfHistBins - 1)
        return fail(HHG_EINVAL, "%s: corrected scores leave the histogram range", who);
      cut = b - kPfHistBias; take_eq = 1; n_b[q] = h[b]; want_eq[q] = need - above;
    }
    n_a[q] = above;
    cuts[q] = PfCut{cut, take_eq, (int)tot_a, (int)tot_b};
    off[q] = (int32_t)std::min<long long>(total, INT_MAX);
    tot_a += n_a[q]; tot_b += n_b[q]; total += n_a[q] + want_eq[q];
  }
  off[nq] = (int32_t)std::min<long long>(total, INT_MAX);
  if (total > cap) return fail(HHG_EINVAL, "%s: %lld survivors exceed the output capacity %d", who, total, cap);
  const size_t n_words = (size_t)(2 * tot_a + tot_b);     // [ids of lists A | their scores | ids of lists B]
  CK(ctx->pf_ids_a.ensure(std::max<size_t>(n_words, 1)));
  CK(ctx->pfb_cuts.ensure(nq));
  CK(cudaMemcpyAsync(ctx->pfb_cuts.p, cuts.data(), (size_t)nq * sizeof(PfCut), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(counters, 0, (size_t)nq * 8, ctx->stream));
  int* d_ids_a = ctx->pf_ids_a.p;
  k_pf_compact<<<dim3((n + 255) / 256, nq), 256, 0, ctx->stream>>>(n, ctx->pf_corr.p, ctx->pfb_cuts.p, d_ids_a,
                                                                    d_ids_a + tot_a, d_ids_a + 2 * tot_a, counters);
  ctx->launches++;
  CK(cudaGetLastError());
  std::vector<int32_t> lists(n_words);
  if (n_words) CK(cudaMemcpyAsync(lists.data(), d_ids_a, n_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  auto order_row = [&](int q) -> std::string {
    const int32_t* a = lists.data() + cuts[q].a_off;
    const int32_t* sa = a + tot_a;
    std::vector<int32_t> b(lists.data() + 2 * tot_a + cuts[q].b_off, lists.data() + 2 * tot_a + cuts[q].b_off + n_b[q]);
    std::sort(b.begin(), b.end(), std::greater<int32_t>());        // ties at the cut: larger index first
    b.resize((size_t)want_eq[q]);
    std::vector<std::pair<int32_t, int32_t>> v;                     // (score, index), descending
    v.reserve((size_t)(n_a[q] + want_eq[q]));
    for (long long k = 0; k < n_a[q]; ++k) v.emplace_back(sa[k], a[k]);
    std::sort(v.begin(), v.end(), std::greater<std::pair<int32_t, int32_t>>());
    for (int32_t id : b) v.emplace_back(cuts[q].cut, id);         // below all of list A, already index-descending
    for (size_t k = 0; k < v.size(); ++k) { ids[off[q] + k] = v[k].second; scores[off[q] + k] = v[k].first; }
    return {};
  };
  if (nq == 1) order_row(0);
  else host_for(nq, order_row);
  return HHG_OK;
}

int hhg_prefilter_select(hhg_ctx* ctx, const hhg_csdb* db, int Lq, int bit_factor, int smax_thresh,
                         int min_hits, int32_t* ids, int32_t* scores, int cap, int* n_out) {
  if (!ctx || !db || Lq < 1 || min_hits < 0 || !ids || !scores || cap < 0 || !n_out)
    return fail(HHG_EINVAL, "hhg_prefilter_select: bad argument");
  int32_t off[2] = {0, 0};
  const int rc = select_rows(ctx, db, 1, &Lq, db->scores.p, bit_factor, smax_thresh, min_hits, ids, scores, cap, off,
                             "hhg_prefilter_select");
  *n_out = off[1];
  return rc;
}

int hhg_prefilter_fetch(hhg_ctx* ctx, const hhg_csdb* db, int32_t* scores) {
  if (!ctx || !db || !scores) return fail(HHG_EINVAL, "hhg_prefilter_fetch: bad argument");
  CK(cudaMemcpyAsync(scores, db->scores.p, (size_t)db->n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

int hhg_prefilter_ungapped(hhg_ctx* ctx, const hhg_csdb* db, int Lq, const uint8_t* prof, int offset,
                           int32_t* scores) {
  int rc = hhg_prefilter_ungapped_run(ctx, db, Lq, prof, offset, 1);
  if (rc != HHG_OK) return rc;
  return hhg_prefilter_fetch(ctx, db, scores);
}

// ------------------------------------------------------------------------------------ prefilter, query batch
// Ungapped stage for nq queries (k_pf_ungapped_batch), planned by pf_plan_batch: memory waves within the context's
// budget (max_bt_bytes, HHG_MAX_BT_GB), one launch per tile round of a wave.
int hhg_prefilter_ungapped_batch_run(hhg_ctx* ctx, const hhg_csdb* db, int nq, const int32_t* Lq,
                                     const uint8_t* const* prof, int offset) {
  if (!ctx || !db || nq < 1 || nq > 65535 || !Lq || !prof || offset < 0 || offset > 255)
    return fail(HHG_EINVAL, "hhg_prefilter_ungapped_batch_run: bad argument");
  for (int q = 0; q < nq; ++q) {
    if (Lq[q] < 1) return fail(HHG_EINVAL, "hhg_prefilter_ungapped_batch_run: query %d has length %d", q, Lq[q]);
    if (!prof[q]) return fail(HHG_EINVAL, "hhg_prefilter_ungapped_batch_run: profile of query %d is NULL", q);
  }
  const int n = db->n;
  const int max_nq = hhg_prefilter_batch_max_queries(ctx, db);
  if (nq > max_nq)
    return fail(HHG_EINVAL, "hhg_prefilter_ungapped_batch_run: %d queries exceed the %d whose scores fit the context's "
                "memory budget (HHG_MAX_BT_GB); split the batch", nq, max_nq);
  CK(cudaSetDevice(ctx->device));
  ctx->pfb_nq = 0;                                  // no valid batch scores until this run is launched
  // the edge slots of the long queries get what the score rows leave of the budget (at least one query per wave)
  const double score_bytes = (double)nq * n * kPfBatchScoreBytes;
  const PfBatchPlan plan = pf_plan_batch(nq, Lq, db->total, std::max(0.0, (double)ctx->max_bt_bytes - score_bytes));
  std::vector<uint32_t> words(plan.slabs.size() * (size_t)kPfSlabWords);
  auto pack = [&](int s) -> std::string {
    pf_pack_slab(plan, s, Lq, prof, offset, words.data() + (size_t)s * kPfSlabWords);
    return {};
  };
  if (plan.slabs.size() == 1) pack(0);
  else host_for((int)plan.slabs.size(), pack);
  CK(ctx->pf_prof.ensure(words.size() * 4));
  CK(ctx->pfb_slabs.ensure(plan.slabs.size()));
  CK(ctx->pfb_scores.ensure((size_t)nq * n));
  CK(ctx->pf_counter.ensure(plan.launches.size()));
  if (plan.max_slots) {
    CK(ctx->pf_edge[0].ensure((size_t)plan.max_slots * db->total));
    CK(ctx->pf_edge[1].ensure((size_t)plan.max_slots * db->total));
  }
  CK(cudaMemcpyAsync(ctx->pf_prof.p, words.data(), words.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->pfb_slabs.p, plan.slabs.data(), plan.slabs.size() * sizeof(PfSlab), cudaMemcpyHostToDevice,
                     ctx->stream));
  CK(cudaMemsetAsync(ctx->pf_counter.p, 0, 4 * plan.launches.size(), ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));           // `words` is a host temporary
  CK(cudaFuncSetAttribute(k_pf_ungapped_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, kPfBatchSmem));
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_pf_ungapped_batch, 512, kPfBatchSmem));
  if (per_sm < 1) return fail(HHG_ECUDA, "prefilter batch kernel does not fit on an SM");
  const long long ctas = (long long)ctx->sm_count * per_sm;
  for (size_t k = 0; k < plan.launches.size(); ++k) {
    const PfLaunch& la = plan.launches[k];
    PfBatchParams P{};
    P.n = n; P.L = db->dL.p; P.off = db->doff.p; P.seq = db->seq.p;
    P.prof32 = reinterpret_cast<const uint32_t*>(ctx->pf_prof.p) + (size_t)la.slab0 * kPfSlabWords;
    P.slabs = ctx->pfb_slabs.p + la.slab0;
    P.nslab = la.nslab;
    P.chunk = pf_chunk(n, la.nslab, ctas);
    P.nchunk = (n + P.chunk - 1) / P.chunk;
    P.offset = offset;
    P.total = db->total;
    P.edge_in = plan.max_slots ? ctx->pf_edge[(la.round + 1) & 1].p : nullptr;
    P.edge_out = plan.max_slots ? ctx->pf_edge[la.round & 1].p : nullptr;
    P.scores = ctx->pfb_scores.p;
    P.counter = ctx->pf_counter.p + k;
    const int grid = (int)std::min<long long>(ctas, (long long)P.nslab * P.nchunk);
    k_pf_ungapped_batch<<<grid, 512, kPfBatchSmem, ctx->stream>>>(P);
    ctx->launches++;
    CK(cudaGetLastError());
  }
  ctx->pfb_nq = nq;
  ctx->pfb_db_serial = db->serial;
  return HHG_OK;
}

// Score rows of a batch: the raw scores (hhg_prefilter_ungapped_batch_run) and the corrected scores
// (hhg_prefilter_select_batch), 4 bytes each per query and sequence, within the context's memory budget.
int hhg_prefilter_batch_max_queries(hhg_ctx* ctx, const hhg_csdb* db) {
  if (!ctx || !db) return 0;
  const double per_query = (double)db->n * kPfBatchScoreBytes;
  return (int)std::max(1.0, std::min(65535.0, std::floor((double)ctx->max_bt_bytes / per_query)));
}

static int check_batch_scores(hhg_ctx* ctx, const hhg_csdb* db, const char* who) {
  if (!ctx->pfb_nq || ctx->pfb_db_serial != db->serial)
    return fail(HHG_EINVAL, "%s: no hhg_prefilter_ungapped_batch_run on this shard", who);
  return HHG_OK;
}

int hhg_prefilter_ungapped_batch_fetch(hhg_ctx* ctx, const hhg_csdb* db, int32_t* scores) {
  if (!ctx || !db || !scores) return fail(HHG_EINVAL, "hhg_prefilter_ungapped_batch_fetch: bad argument");
  if (int rc = check_batch_scores(ctx, db, "hhg_prefilter_ungapped_batch_fetch")) return rc;
  CK(cudaSetDevice(ctx->device));
  CK(cudaMemcpyAsync(scores, ctx->pfb_scores.p, (size_t)ctx->pfb_nq * db->n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return HHG_OK;
}

int hhg_prefilter_select_batch(hhg_ctx* ctx, const hhg_csdb* db, int nq, const int32_t* Lq, int bit_factor,
                               int smax_thresh, int min_hits, int32_t* ids, int32_t* scores, int cap, int32_t* off) {
  if (!ctx || !db || nq < 1 || !Lq || min_hits < 0 || !ids || !scores || cap < 0 || !off)
    return fail(HHG_EINVAL, "hhg_prefilter_select_batch: bad argument");
  for (int q = 0; q < nq; ++q)
    if (Lq[q] < 1) return fail(HHG_EINVAL, "hhg_prefilter_select_batch: query %d has length %d", q, Lq[q]);
  if (int rc = check_batch_scores(ctx, db, "hhg_prefilter_select_batch")) return rc;
  if (nq != ctx->pfb_nq)
    return fail(HHG_EINVAL, "hhg_prefilter_select_batch: %d queries, the last batch run had %d", nq, ctx->pfb_nq);
  return select_rows(ctx, db, nq, Lq, ctx->pfb_scores.p, bit_factor, smax_thresh, min_hits, ids, scores, cap, off,
                     "hhg_prefilter_select_batch");
}

// Gapped stage 2 for the requests of nq queries in one k_prefilter_sw_batch launch: request r scores query
// req_query[r] against sequence ids[r].  A query's striped profile is staged in shared memory when it fits next to
// its own working columns (the rule of hhg_prefilter_sw), else it is read from L2.
int hhg_prefilter_sw_batch(hhg_ctx* ctx, const hhg_csdb* db, int nq, const int32_t* Lq, const uint8_t* const* prof,
                           int n, const int32_t* req_query, const int32_t* ids, int gap_open, int gap_extend, int bias,
                           int32_t* scores) {
  if (!ctx || !db || nq < 1 || !Lq || !prof || n < 0 || (n > 0 && (!req_query || !ids || !scores)))
    return fail(HHG_EINVAL, "hhg_prefilter_sw_batch: bad argument");
  const size_t kSmemMax = 227 * 1024;
  int Wmax = 0;
  for (int q = 0; q < nq; ++q) {
    if (Lq[q] < 1) return fail(HHG_EINVAL, "hhg_prefilter_sw_batch: query %d has length %d", q, Lq[q]);
    if (!prof[q]) return fail(HHG_EINVAL, "hhg_prefilter_sw_batch: profile of query %d is NULL", q);
    Wmax = std::max(Wmax, (Lq[q] + 31) / 32);
  }
  const size_t work_bytes = (size_t)8 * 3 * Wmax * 32;           // H/H/E columns of the 8 warps of a CTA
  if (work_bytes > kSmemMax)
    return fail(HHG_EINVAL, "prefilter sw: query length %d too long (working columns exceed shared memory)", Wmax * 32);
  for (int r = 0; r < n; ++r) {
    if (req_query[r] < 0 || req_query[r] >= nq) return fail(HHG_EINVAL, "prefilter sw batch: request %d: query %d out of range", r, req_query[r]);
    if (ids[r] < 0 || ids[r] >= db->n) return fail(HHG_EINVAL, "prefilter sw batch: request %d: id %d out of range", r, ids[r]);
  }
  if (n == 0) return HHG_OK;
  CK(cudaSetDevice(ctx->device));
  // requests grouped by query (stable), one striped profile per query that has requests
  std::vector<int> first(nq + 1, 0);
  for (int r = 0; r < n; ++r) ++first[req_query[r] + 1];
  for (int q = 0; q < nq; ++q) first[q + 1] += first[q];
  std::vector<int> order(n), grouped_ids(n);
  {
    std::vector<int> fill(first.begin(), first.end() - 1);
    for (int r = 0; r < n; ++r) { const int k = fill[req_query[r]]++; order[k] = r; grouped_ids[k] = ids[r]; }
  }
  // shared memory per query as hhg_prefilter_sw lays it out: [striped profile, if it fits][working columns]
  std::vector<SwBatchQuery> qs(nq);
  size_t prof_total = 0, ctrl_off = 0;
  for (int q = 0; q < nq; ++q) {
    const int W = (Lq[q] + 31) / 32;
    const size_t bytes = (size_t)220 * W * 32, work = (size_t)8 * 3 * W * 32;
    qs[q].W = W;
    qs[q].smem = bytes + work <= kSmemMax;
    qs[q].work_off = qs[q].smem ? (int)bytes : 0;
    qs[q].prof_off = -1;
    if (first[q + 1] == first[q]) continue;
    qs[q].prof_off = (long long)prof_total;
    prof_total += bytes;
    ctrl_off = std::max(ctrl_off, (size_t)qs[q].work_off + work);
  }
  ctrl_off = (ctrl_off + 15) & ~(size_t)15;
  std::vector<uint8_t> striped(prof_total);
  for (int q = 0; q < nq; ++q) {
    if (qs[q].prof_off < 0) continue;
    const int W = qs[q].W;
    uint8_t* out = striped.data() + qs[q].prof_off;
    for (int k = 0; k < 220; ++k)
      for (int j = 0; j < W; ++j)
        for (int l = 0; l < 32; ++l) {
          const int pos = l * W + j;
          out[((size_t)k * W + j) * 32 + l] = pos < Lq[q] ? prof[q][(size_t)k * Lq[q] + pos] : (uint8_t)bias;
        }
  }
  const int kChunk = 64;                                           // requests per work item
  std::vector<int4> items;
  for (int q = 0; q < nq; ++q)
    for (int r0 = first[q]; r0 < first[q + 1]; r0 += kChunk) items.push_back(make_int4(q, r0, std::min(kChunk, first[q + 1] - r0), 0));
  CK(ctx->sw_prof.ensure(prof_total)); CK(ctx->sw_ids.ensure(n)); CK(ctx->sw_scores.ensure(n));
  CK(ctx->swb_items.ensure(items.size())); CK(ctx->swb_queries.ensure(nq)); CK(ctx->pf_counter.ensure(1));
  CK(cudaMemcpyAsync(ctx->sw_prof.p, striped.data(), prof_total, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->sw_ids.p, grouped_ids.data(), (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->swb_items.p, items.data(), items.size() * sizeof(int4), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->swb_queries.p, qs.data(), (size_t)nq * sizeof(SwBatchQuery), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->pf_counter.p, 0, 4, ctx->stream));
  SwBatchParams P{};
  P.nitem = (int)items.size(); P.items = ctx->swb_items.p; P.queries = ctx->swb_queries.p; P.ids = ctx->sw_ids.p;
  P.L = db->dL.p; P.off = db->doff.p; P.seq = db->seq.p; P.prof = ctx->sw_prof.p;
  P.ctrl_off = (int)ctrl_off;
  P.gap_open = gap_open; P.gap_extend = gap_extend; P.bias = bias;
  P.scores = ctx->sw_scores.p; P.counter = ctx->pf_counter.p;
  const size_t smem = ctrl_off + 16;
  CK(cudaFuncSetAttribute(k_prefilter_sw_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_prefilter_sw_batch, 256, smem));
  if (per_sm < 1) return fail(HHG_ECUDA, "prefilter sw batch kernel does not fit on an SM");
  const int grid = (int)std::min<long long>((long long)ctx->sm_count * per_sm, (long long)items.size());
  k_prefilter_sw_batch<<<grid, 256, smem, ctx->stream>>>(P);
  ctx->launches++;
  CK(cudaGetLastError());
  std::vector<int32_t> got(n);
  CK(cudaMemcpyAsync(got.data(), ctx->sw_scores.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (int k = 0; k < n; ++k) scores[order[k]] = got[k];
  return HHG_OK;
}
