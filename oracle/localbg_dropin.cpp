// oracle/localbg_dropin.cpp -- TEST INFRASTRUCTURE: the drop-in check (oracle/ref_gpu_adapter.cpp, compiled unchanged
// into this binary) with the column-score options of the reference's CLIs.
//
// usage: hh_dropin_check_localbg [--sc N] [--scwin D] <arguments of hh_dropin_check>
//   --sc N     par.columnscore = N (-sc; 5 = local amino-acid composition correction of query and templates)
//   --scwin D  par.half_window_size_local_aa_bg_freqs = max(1, D) and par.columnscore = 5 (-scwin, as hhblits,
//              hhsearch and hhalign parse it: src/hhblits.cpp:766-771)
//
// Both sides of the check read the options from the Parameters object the drop-in check constructs: every Parameters
// made in the included source is an ScParameters, which applies them in its constructor, before PrepareQueryHMM and
// the reference's runner see it.  The adapter's call to hhg_db_apply_null_model is preceded by hhg_set_scwin with
// that object's half window, which is what a binding of the library does (INTEGRATION.md section 2).  Built by
// oracle/localbg_ref.mk into oracle/_ref/hh_dropin_check_localbg.

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <map>
#include <set>
#include <memory>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

// every reference header the drop-in check includes, with its test-harness access, before Parameters is renamed below
#define private public
#define protected public
#include "hhdecl.h"
#include "hhhmm.h"
#include "hhhmmsimd.h"
#include "hhviterbi.h"
#include "hhviterbimatrix.h"
#include "hhviterbirunner.h"
#include "hhmatrices.h"
#include "hhfunc.h"
#include "hhdatabase.h"
#include "hhhit.h"
#include "hhposteriordecoder.h"
#include "hhposteriordecoderrunner.h"
#include "hhposteriormatrix.h"
#include "hhprefilter.h"
#include "ffindexdatabase.h"
#include "hash.h"
#include "cs219.lib.h"
#undef private
#undef protected

#include "../include/hhg.h"

namespace {
int g_columnscore = -1;   // -1: the reference's default
int g_scwin = 0;          // 0: the reference's default
}  // namespace

struct ScParameters : Parameters {
  ScParameters(const int argc, const char** argv) : Parameters(argc, argv) {
    if (g_columnscore >= 0) columnscore = g_columnscore;
    if (g_scwin > 0) half_window_size_local_aa_bg_freqs = g_scwin;
    printf("hh_dropin_check_localbg: column score %d, half window %d\n", columnscore, half_window_size_local_aa_bg_freqs);
  }
};

#define Parameters ScParameters
#define hhg_db_apply_null_model(ctx, db, q_pav, pb, cs) \
  (hhg_set_scwin((ctx), par.half_window_size_local_aa_bg_freqs), ::hhg_db_apply_null_model((ctx), (db), (q_pav), (pb), (cs)))
#define main hh_dropin_check_main
#include "ref_gpu_adapter.cpp"
#undef main
#undef hhg_db_apply_null_model
#undef Parameters

int main(int argc, char** argv) {
  std::vector<char*> args(argv, argv + argc);
  for (size_t k = 1; k + 1 < args.size();) {
    if (!strcmp(args[k], "--sc")) {
      g_columnscore = atoi(args[k + 1]);
    } else if (!strcmp(args[k], "--scwin")) {
      g_scwin = std::max(1, atoi(args[k + 1]));
      g_columnscore = 5;
    } else {
      ++k;
      continue;
    }
    args.erase(args.begin() + k, args.begin() + k + 2);
  }
  args.push_back(nullptr);
  return hh_dropin_check_main((int)args.size() - 1, args.data());
}
