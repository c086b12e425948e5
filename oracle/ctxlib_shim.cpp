// oracle/ctxlib_shim.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A C-ABI driver around the UNMODIFIED reference's generative context-library engine (the branch of
// InitializePseudocountsEngine, src/hhfunc.cpp:229-236, that `-contxt <file>` takes for any file that is not a .crf):
// cs::ContextLibrary's reader, TransformToLog, cs::LibraryPseudocounts, HMM::AddContextSpecificPseudocounts and
// CalculateAminoAcidBackground.  Built by oracle/ctxlib_ref.mk into oracle/_ref/libhhref_ctxlib.so against the same
// reference objects as oracle/ref_shim.cpp, with data/context_data.lib embedded.  Tests load it through
// oracle/ctxlib_binding.py; nothing here is linked into the product library.
//
// This file contains no reference code: it includes the reference headers at build time and calls their API.  The
// HMM's frequency arrays are reached with the test-harness trick of oracle/ref_shim.cpp (#define private public after
// the std headers).

#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <iostream>
#include <map>
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
#include "context_library-inl.h"
#include "library_pseudocounts-inl.h"
#undef private
#undef protected

extern "C" const unsigned char _binary_context_data_lib_start[];
extern "C" const unsigned char _binary_context_data_lib_end[];

namespace {

struct LibCtx {
  Parameters* par = nullptr;
  float pb[21] __attribute__((aligned(32)));
  float P[20][20] __attribute__((aligned(32)));
  float R[20][20] __attribute__((aligned(32)));
  float S[20][20] __attribute__((aligned(32)));
  float Sim[20][20] __attribute__((aligned(32)));
};
LibCtx* g = nullptr;
const char* kArgv[] = {"hhblits"};

void init() {
  if (g) return;
  Log::reporting_level() = WARNING;
  g = new LibCtx();
  g->par = new Parameters(1, kArgv);
  SetSubstitutionMatrix(g->par->matrix, g->pb, g->P, g->R, g->S, g->Sim);
}

// A context library given as text, read by cs::ContextLibrary's own reader through fmemopen and transformed to log
// space, as InitializePseudocountsEngine does.  Cached by content; a refused text is cached with the reader's message.
struct LibByText {
  std::string text, err;
  std::unique_ptr<cs::ContextLibrary<cs::AA>> lib;
};
std::vector<std::unique_ptr<LibByText>> g_libs;
std::string g_err;

const cs::ContextLibrary<cs::AA>* lib_from_text(const char* text, long long len) {
  for (auto& e : g_libs)
    if ((long long)e->text.size() == len && memcmp(e->text.data(), text, (size_t)len) == 0) {
      g_err = e->err;
      return e->lib.get();
    }
  std::unique_ptr<LibByText> e(new LibByText());
  e->text.assign(text, (size_t)len);
  FILE* fin = fmemopen((void*)e->text.data(), e->text.size(), "r");
  try {
    e->lib.reset(new cs::ContextLibrary<cs::AA>(fin));
    cs::TransformToLog(*e->lib);
  } catch (const std::exception& ex) {        // cs::Exception, what the reader throws
    e->lib.reset();
    e->err = ex.what();
    if (e->err.empty()) e->err = "refused";
  }
  fclose(fin);
  if (g_libs.size() >= 16) g_libs.erase(g_libs.begin());
  g_libs.push_back(std::move(e));
  g_err = g_libs.back()->err;
  return g_libs.back()->lib.get();
}

// HMM::AddContextSpecificPseudocounts + CalculateAminoAcidBackground on an HMM holding f[(L+2)*20] and Neff_M[L+1]
void run_engine(cs::Pseudocounts<cs::AA>* engine, cs::Admix* mode, int L, const float* f, const float* neff_m,
                float neff_hmm, float* p, float* pav) {
  std::unique_ptr<HMM> h(new HMM(MAXSEQDIS, L + 2));
  h->L = L;
  h->has_pseudocounts = false;
  h->Neff_HMM = neff_hmm;
  for (int i = 0; i <= L + 1; ++i) for (int a = 0; a < 20; ++a) h->f[i][a] = f[(size_t)i * 20 + a];
  for (int i = 0; i <= L; ++i) h->Neff_M[i] = neff_m[i];
  h->AddContextSpecificPseudocounts(engine, mode);
  h->CalculateAminoAcidBackground(g->pb);
  for (int i = 0; i <= L + 1; ++i) for (int a = 0; a < 20; ++a) p[(size_t)i * 20 + a] = h->p[i][a];
  for (int a = 0; a < 20; ++a) pav[a] = h->pav[a];
}

}  // namespace

extern "C" {

// the embedded data/context_data.lib, so tests can hand it to the product without reading the reference tree
const unsigned char* hhref_lib_text(long long* len) {
  *len = (long long)(_binary_context_data_lib_end - _binary_context_data_lib_start);
  return _binary_context_data_lib_start;
}

// the background CalculateAminoAcidBackground reads: SetSubstitutionMatrix's until hhref_lib_set_pb replaces it (in
// hhblits an HHM file read earlier overwrites it, src/hhhmm.cpp:543)
void hhref_lib_pb(float* out) { init(); memcpy(out, g->pb, 20 * sizeof(float)); }
void hhref_lib_set_pb(const float* pb) { init(); memcpy(g->pb, pb, 20 * sizeof(float)); }

// the message of the last refused text (empty when it was accepted)
const char* hhref_lib_error() { return g_err.c_str(); }

// Profile k of the library in `text` after TransformToLog: *wlen, log prior, probs[wlen*20] (log space; may be NULL)
// and pc[20] (the central column in linear space).  Returns the number of profiles, -1 when the reader refused the
// text (hhref_lib_error), -2 when k is out of range.
int hhref_lib_text_state(const char* text, long long len, int k, int* wlen, double* prior, double* probs, double* pc) {
  const cs::ContextLibrary<cs::AA>* lib = lib_from_text(text, len);
  if (!lib) return -1;
  if (k < 0 || k >= (int)lib->size()) return -2;
  const cs::ContextProfile<cs::AA>& s = (*lib)[k];
  *wlen = (int)s.probs.length();
  *prior = s.prior;
  if (probs)
    for (size_t j = 0; j < s.probs.length(); ++j)
      for (int a = 0; a < 20; ++a) probs[j * 20 + a] = s.probs[j][a];
  for (int a = 0; a < 20; ++a) pc[a] = s.pc[a];
  return (int)lib->size();
}

// cs::LibraryPseudocounts(lib, csw, csb) on the library in `text` with one of cs::ConstantAdmix(pca) ("constant"),
// cs::CSBlastAdmix(pca, pcb) ("csblast") or cs::HHsearchAdmix(pca, pcb, pcc) ("hhsearch"), then
// HMM::AddContextSpecificPseudocounts + CalculateAminoAcidBackground.  csw and csb are the doubles the engine gets
// (hhblits passes its float par.csw / par.csb).  Returns L, -1 when the reader refused the text, -2 for an unknown
// admixture class.
int hhref_context_pc_lib(const char* text, long long len, double csw, double csb, const char* admix, double pca,
                         double pcb, double pcc, int L, const float* f, const float* neff_m, float neff_hmm, float* p,
                         float* pav) {
  init();
  const cs::ContextLibrary<cs::AA>* lib = lib_from_text(text, len);
  if (!lib) return -1;
  std::unique_ptr<cs::Admix> mode;
  if (!strcmp(admix, "constant")) mode.reset(new cs::ConstantAdmix(pca));
  else if (!strcmp(admix, "csblast")) mode.reset(new cs::CSBlastAdmix(pca, pcb));
  else if (!strcmp(admix, "hhsearch")) mode.reset(new cs::HHsearchAdmix(pca, pcb, pcc));
  else return -2;
  cs::LibraryPseudocounts<cs::AA> engine(*lib, csw, csb);
  run_engine(&engine, mode.get(), L, f, neff_m, neff_hmm, p, pav);
  return L;
}

// The reference's own dispatch: InitializePseudocountsEngine with par.clusterfile = path (a file whose extension is
// not "crf") and par.csw / par.csb, then the engine of the query HMM (engine 0) or of the prefilter profile (1) with
// the admixture par gives it.  Returns L, -1 when no context library engine was built.
int hhref_context_pc_dispatch(const char* path, float csw, float csb, int engine, int L, const float* f,
                              const float* neff_m, float neff_hmm, float* p, float* pav) {
  init();
  g->par->clusterfile = path;
  g->par->csw = csw;
  g->par->csb = csb;
  cs::ContextLibrary<cs::AA>* context_lib = nullptr;
  cs::Crf<cs::AA>* crf = nullptr;
  cs::Pseudocounts<cs::AA>* e[2] = {nullptr, nullptr};
  cs::Admix* m[2] = {nullptr, nullptr};
  InitializePseudocountsEngine(*g->par, context_lib, crf, e[0], m[0], e[1], m[1]);
  const int rc = context_lib && !crf ? L : -1;
  if (rc == L) run_engine(e[engine ? 1 : 0], m[engine ? 1 : 0], L, f, neff_m, neff_hmm, p, pav);
  DeletePseudocountsEngine(context_lib, crf, e[0], m[0], e[1], m[1]);
  return rc;
}

}  // extern "C"
