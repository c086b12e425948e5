// tests/emul/stage_cache_emul.cpp -- C entry points over the product's staged-shard bookkeeping
// (hh-suite_b200/csrc/hhg_stage_cache.h, unmodified), so tests/test_staged_cache_cpu.py drives it without a device.
#include "../../hh-suite_b200/csrc/hhg_stage_cache.h"

using hhg::StageCache;
using hhg::StageItem;
using hhg::StageStats;

extern "C" {

void* sc_create(int slots, long long cols) { return new StageCache(slots, cols); }
void sc_destroy(void* c) { delete static_cast<StageCache*>(c); }

// StageCache::request; items_out[5 * k ..] = {src, dst, len, slot, global} of copy k (capacity n), freed_out[n_freed]
// (capacity: the number of slots).  out[6] = {hits, copied, bytes, evicted, n_items, n_freed} or, on failure,
// out[0..2] = {bad position, slots needed, columns needed}.
int sc_request(void* c, int n, const int32_t* ids, int n_store, const int32_t* L, const long long* src_off,
               int32_t* local, long long* items_out, int32_t* freed_out, long long* out) {
  std::vector<StageItem> items;
  std::vector<int> freed;
  StageStats st{};
  int bad = -1;
  long long need_slots = 0, need_cols = 0;
  const int rc = static_cast<StageCache*>(c)->request(n, ids, n_store, L, src_off, local, &items, &freed, &st, &bad,
                                                      &need_slots, &need_cols);
  if (rc != 0) {
    out[0] = bad; out[1] = need_slots; out[2] = need_cols;
    return rc;
  }
  for (size_t k = 0; k < items.size(); ++k) {
    const StageItem& it = items[k];
    long long* o = items_out + 5 * k;
    o[0] = it.src; o[1] = it.dst; o[2] = it.len; o[3] = it.slot; o[4] = it.global;
  }
  for (size_t k = 0; k < freed.size(); ++k) freed_out[k] = freed[k];
  out[0] = st.hits; out[1] = st.copied; out[2] = st.bytes; out[3] = st.evicted;
  out[4] = (long long)items.size(); out[5] = (long long)freed.size();
  return 0;
}

// slot -> {global id or -1, first arena record, length}
void sc_slot(void* c, int s, long long* out) {
  const StageCache* sc = static_cast<StageCache*>(c);
  out[0] = sc->global_of(s); out[1] = sc->off_of(s); out[2] = sc->len_of(s);
}
int sc_resident(void* c) { return static_cast<StageCache*>(c)->resident(); }

}  // extern "C"
