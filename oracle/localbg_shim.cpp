// oracle/localbg_shim.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A C-ABI driver around the UNMODIFIED reference's local amino-acid composition correction (-sc 5 / -scwin D):
// HMM::DivideBySqrtOfLocalBackgroundFreqs (src/hhhmm.cpp:1979-2035) on a caller's profile, PrepareQueryHMM under
// par.columnscore = 5 (src/hhfunc.cpp:121-160) and the steps of PrepareTemplateHMM with IncludeNullModelInHMM case 5
// (src/hhfunc.cpp:165-202, src/hhhmm.cpp:2095-2103).  Built by oracle/localbg_ref.mk into
// oracle/_ref/libhhref_localbg.so against the same reference objects as oracle/ref_shim.cpp.  Tests load it through
// oracle/localbg_binding.py; nothing here is linked into the product library.
//
// This file contains no reference code: it includes the reference headers at build time and calls their API.  The
// HMM's arrays are reached with the test-harness trick of oracle/ref_shim.cpp (#define private public after the std
// headers).

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

#define private public
#define protected public
#include "hhdecl.h"
#include "hhhmm.h"
#include "hhmatrices.h"
#include "hhfunc.h"
#undef private
#undef protected

namespace {

struct LbCtx {
  Parameters* par = nullptr;
  float pb[21] __attribute__((aligned(32)));
  float P[20][20] __attribute__((aligned(32)));
  float R[20][20] __attribute__((aligned(32)));
  float S[20][20] __attribute__((aligned(32)));
  float Sim[20][20] __attribute__((aligned(32)));
  HMM* q = nullptr;   // the last query prepared by hhlb_prepare_query_hhm
};
LbCtx* g = nullptr;
const char* kArgv[] = {"hhblits"};
constexpr int kMaxres = 4096;   // HMM capacity of the file readers below (the shim's usual value)

void init() {
  if (g) return;
  Log::reporting_level() = WARNING;
  g = new LbCtx();
  g->par = new Parameters(1, kArgv);
  g->par->nocontxt = 1;
  g->par->maxres = kMaxres;
  SetSubstitutionMatrix(g->par->matrix, g->pb, g->P, g->R, g->S, g->Sim);
  g->q = new HMM(MAXSEQDIS, kMaxres);
}

// HMM::Read of an HHM file into h; the background pb is set to the file's NULL line, as the reader does.
bool read_hhm(const char* path, HMM* h) {
  FILE* f = fopen(path, "r");
  if (!f) return false;
  char pathbuf[NAMELEN];
  Pathname(pathbuf, const_cast<char*>(path));
  h->Read(f, g->par->maxcol, g->par->nseqdis, g->pb, pathbuf);
  fclose(f);
  return true;
}

void export_p(const HMM* h, float* p) {
  for (int i = 0; i <= h->L + 1; ++i)
    for (int a = 0; a < 20; ++a) p[(size_t)i * 20 + a] = h->p[i][a];
}

}  // namespace

extern "C" {

// HMM::DivideBySqrtOfLocalBackgroundFreqs(D, pb) on p_in[(L+2)*20] -> p_out[(L+2)*20], on an HMM allocated for this L.
// The routine computes 2*D+1 in int, which overflows for D >= 2^30; every D >= 16383 takes its whole-profile branch
// for L <= 32767, where D plays no further part, so such D are passed as 16383.  Returns L, or -1 for L outside
// [1, 32767].
int hhlb_local_bg(int L, const float* p_in, const float* pb, int D, float* p_out) {
  if (L < 1 || L > 32767) return -1;
  init();
  HMM* h = new HMM(MAXSEQDIS, L + 2);
  h->L = L;
  for (int i = 0; i <= L + 1; ++i)
    for (int a = 0; a < 20; ++a) h->p[i][a] = p_in[(size_t)i * 20 + a];
  h->divided_by_local_bg_freqs = false;
  h->DivideBySqrtOfLocalBackgroundFreqs(std::min(D, 16383), pb);
  export_p(h, p_out);
  delete h;
  return L;
}

// Read an HHM query and run PrepareQueryHMM (nocontxt branch) with par.columnscore = columnscore and
// par.half_window_size_local_aa_bg_freqs = D.  p[(L_cap+2)*20] receives HMM::p, pb_out[20] the background the
// reader set.  The prepared query stays for hhlb_prepare_template_hhm.  Returns L, -1 without the file, -2 when
// L > L_cap.
int hhlb_prepare_query_hhm(const char* path, int columnscore, int D, int L_cap, float* p, float* pb_out) {
  init();
  if (!read_hhm(path, g->q)) return -1;
  if (g->q->L > L_cap) return -2;
  Parameters& par = *g->par;
  par.columnscore = columnscore;
  par.half_window_size_local_aa_bg_freqs = D;
  char input_format = 0;
  PrepareQueryHMM(par, input_format, g->q, nullptr, nullptr, g->pb, g->R);
  export_p(g->q, p);
  memcpy(pb_out, g->pb, 20 * sizeof(float));
  return g->q->L;
}

// Read an HHM template and run the steps of PrepareTemplateHMM (src/hhfunc.cpp:165-202) one by one, exporting HMM::p
// before (p_raw) and after (p_prep) IncludeNullModelInHMM with par.columnscore of the last hhlb_prepare_query_hhm
// call (5 needs that query to have been divided).  pb_out[20]: the background the reader set.  Returns L, -1 without
// the file, -2 when L > L_cap.
int hhlb_prepare_template_hhm(const char* path, int L_cap, float* p_raw, float* p_prep, float* pb_out) {
  init();
  HMM* t = new HMM(MAXSEQDIS, kMaxres);
  if (!read_hhm(path, t)) { delete t; return -1; }
  const int L = t->L;
  if (L > L_cap) { delete t; return -2; }
  Parameters& par = *g->par;
  t->AddTransitionPseudocounts(par.gapd, par.gape, par.gapf, par.gapg, par.gaph, par.gapi, par.gapb, par.gapb);
  t->PreparePseudocounts(g->R);
  t->AddAminoAcidPseudocounts(par.pc_hhm_nocontext_mode, par.pc_hhm_nocontext_a, par.pc_hhm_nocontext_b,
                              par.pc_hhm_nocontext_c);
  t->CalculateAminoAcidBackground(g->pb);
  export_p(t, p_raw);
  t->IncludeNullModelInHMM(g->q, t, par.columnscore, par.half_window_size_local_aa_bg_freqs, g->pb);
  export_p(t, p_prep);
  memcpy(pb_out, g->pb, 20 * sizeof(float));
  delete t;
  return L;
}

// The pseudocount matrix R[a][b] of SetSubstitutionMatrix (the R the loaders take), out[400].
void hhlb_get_R(float* out) {
  init();
  memcpy(out, g->R, 400 * sizeof(float));
}

}  // extern "C"
