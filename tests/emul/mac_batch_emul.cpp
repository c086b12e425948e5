// tests/emul/mac_batch_emul.cpp -- TEST INFRASTRUCTURE: runs the product's MAC kernels (hh-suite_b200/csrc/hhg_mac.cuh,
// unmodified source) on the CPU through tests/emul/cuda_emul.h with a batch of queries in one launch (MacArgs.req_q,
// the layout hhg_mac_realign_batch builds).  Built by tests/test_mac_batch_emul_cpu.py:
//   g++ -O1 -std=c++20 -ffp-contract=off -fPIC -shared -pthread -o tests/emul/libmacbatchemul.so tests/emul/mac_batch_emul.cpp
#include "cuda_emul.h"

#include <cfloat>

namespace hhg {
struct alignas(16) ColRec {   // as in hh-suite_b200/csrc/hhg_kernels.cuh
  float p[20];
  float m2m, m2d, d2m, d2d, i2m, i2i, m2i;
  uint32_t ss;
};
static_assert(sizeof(ColRec) == 112, "ColRec");
}  // namespace hhg

namespace hhg {
alignas(16) unsigned char mac_smem[256 * 1024];   // the block's dynamic shared memory (blocks run one at a time)
}

#include "../../hh-suite_b200/csrc/hhg_mac.cuh"

using namespace hhg;

static void reset_query_rows(float* tr, int L) {     // initializeQueryHMMTransitions, as hhg_mac_query_set_batch does
  tr[1] = tr[2] = tr[3] = tr[4] = tr[5] = tr[6] = 0.f;
  float* e = tr + (size_t)L * 7; e[0] = 1.f; e[1] = e[2] = e[3] = e[4] = 0.f; e[5] = 1.f; e[6] = 0.f;
}
static void reset_template_rows(float* tr, int L) {  // initializeForAlignment, as hhg_mac_realign_batch does
  tr[0] = 1.f; tr[1] = tr[2] = tr[3] = tr[4] = tr[5] = tr[6] = 0.f;
  float* e = tr + (size_t)L * 7; e[0] = 1.f; e[1] = e[2] = e[3] = e[4] = 0.f; e[5] = 1.f; e[6] = 0.f;
}

// nq queries (q_p: (Lq+2)*20 floats each, q_tr_lin: (Lq+1)*7 each, concatenated) and n requests in one k_mac_band and
// one k_mac_realign launch: request r = query req_q[r] against its own prepared template (t_p: (Lt+2)*20, t_tr_lin:
// (Lt+1)*7, concatenated in request order).  Request r's path is written at sum_{s<r}(Lq_s + Lt_s + 2) of out_*, its
// posterior matrix at sum_{s<r}(Lq_s+1)(Lt_s+1) of post; hits: n MacHitOut records.  Returns 0.
extern "C" int emul_mac_realign_batch(int nq, const int* qL, const float* q_p, const float* q_tr_lin, int n,
                                      const int* req_q, const int* Lt, const float* t_p, const float* t_tr_lin,
                                      const int* vit5, const long long* vit_off, const int* vit_i, const int* vit_j,
                                      int local, double Cshift, float mact, int smem_bytes, int band_scan, void* hits,
                                      int* out_i, int* out_j, uint8_t* out_states, float* out_post, float* post_out) {
  std::vector<long long> q_off(2 * (size_t)nq);
  long long np = 0, ntr = 0;
  for (int q = 0; q < nq; ++q) {
    q_off[q] = np; np += (long long)(qL[q] + 2) * 20;
    q_off[nq + q] = ntr; ntr += (long long)(qL[q] + 1) * 7;
  }
  std::vector<float> qtr(q_tr_lin, q_tr_lin + ntr);
  for (int q = 0; q < nq; ++q) reset_query_rows(qtr.data() + q_off[nq + q], qL[q]);
  std::vector<long long> rec0(n), tr_off(n), cell_off(n), row_off(n), scale_off(n), path_off(n);
  long long nrec = 0, nt = 0, ncell = 0, nrow = 0, nscale = 0, npath = 0, np_t = 0;
  std::vector<ColRec> cols;
  std::vector<float> ttr;
  for (int r = 0; r < n; ++r) {
    const int L = Lt[r], Lq = qL[req_q[r]];
    rec0[r] = nrec; tr_off[r] = nt; cell_off[r] = ncell; row_off[r] = nrow; scale_off[r] = nscale; path_off[r] = npath;
    for (int j = 1; j <= L; ++j) {
      ColRec c{};
      for (int a = 0; a < 20; ++a) c.p[a] = t_p[np_t + (size_t)j * 20 + a];
      cols.push_back(c);
    }
    ttr.insert(ttr.end(), t_tr_lin + nt, t_tr_lin + nt + (long long)(L + 1) * 7);
    reset_template_rows(ttr.data() + nt, L);
    nrec += L; nt += (long long)(L + 1) * 7; np_t += (long long)(L + 2) * 20;
    ncell += (long long)(Lq + 1) * (L + 1);
    nrow += 11LL * (L + 3) + (L + 3 + 7) / 8 + 1;
    nscale += Lq + 3;
    npath += (long long)Lq + L + 2;
  }
  std::vector<float> post((size_t)ncell, 0.f);
  std::vector<uint8_t> off((size_t)ncell, 0), bt((size_t)ncell, 0);
  std::vector<double> rows((size_t)nrow, 0.0), scale((size_t)nscale, 0.0);
  std::vector<MacHitOut> out((size_t)n);
  MacArgs A{};
  A.n = n; A.local = local; A.mact = mact; A.Cshift = Cshift;
  A.q_p = q_p; A.q_tr = qtr.data();
  A.req_q = req_q; A.q_L = qL; A.q_p_off = q_off.data(); A.q_tr_off = q_off.data() + nq; A.scale_off = scale_off.data();
  A.cols = cols.data(); A.rec0 = rec0.data(); A.Lt = Lt; A.t_tr = ttr.data(); A.tr_off = tr_off.data();
  A.vit = vit5; A.vit_off = vit_off; A.vit_i = vit_i; A.vit_j = vit_j;
  A.cell_off = cell_off.data(); A.post = post.data(); A.off = off.data(); A.bt = bt.data();
  A.row_off = row_off.data(); A.rows = rows.data(); A.scale = scale.data(); A.out = out.data();
  A.path_off = path_off.data(); A.out_i = out_i; A.out_j = out_j; A.out_states = out_states; A.out_post = out_post;
  A.smem_rows = smem_bytes;
  A.band_scan = band_scan;
  emul_launch(emul_dim3(n), 256, k_mac_band, A);
  emul_launch(emul_dim3(n), 32, k_mac_realign, A);
  std::memcpy(hits, out.data(), out.size() * sizeof(MacHitOut));
  std::memcpy(post_out, post.data(), post.size() * sizeof(float));
  return 0;
}
