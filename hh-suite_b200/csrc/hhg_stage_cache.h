// hh-suite_b200/csrc/hhg_stage_cache.h -- host bookkeeping of a staged shard (hhg_db_create_staged / hhg_db_stage):
// which targets of the host-resident store occupy which local slot and which run of the device column arena.
// Plain C++, no CUDA: hhg_api.cu drives it and tests/emul/stage_cache_emul.cpp compiles it without a device.
//
// Rules (DESIGN 4.12):
//   * a resident target keeps its slot (= local id) and its arena run until it is evicted;
//   * a missing target takes a free slot and the first free arena run that holds its columns (first fit; freed runs
//     are merged with their free neighbours);
//   * when no slot or no run is free, targets NOT named by the current request are evicted, least recently staged
//     first, until there is one -- the arena is not compacted on this path;
//   * when every other target is gone and the request's own residents still fragment the arena, the request's targets
//     are laid out again from column 0 (slots are kept, all of them are copied again).  So a request fails only when
//     its own distinct targets need more slots or columns than the shard has, and that is checked before anything
//     changes.
#pragma once
#include <cstdint>
#include <map>
#include <set>
#include <unordered_map>
#include <utility>
#include <vector>

namespace hhg {

struct StageItem {          // one target to copy: store records [src, src + len) -> arena records [dst, dst + len)
  long long src, dst;
  int len, slot, global;
};

struct StageStats {         // hhg_stage_stats of include/hhg.h
  long long hits, copied, bytes, evicted;
};

class StageCache {
 public:
  StageCache(int slots, long long cols) : cap_cols_(cols), slot_(slots) {
    for (int s = slots - 1; s >= 0; --s) free_slots_.push_back(s);
    if (cols > 0) free_[0] = cols;
  }
  int slots() const { return (int)slot_.size(); }
  long long cols() const { return cap_cols_; }
  int resident() const { return (int)where_.size(); }
  // slot -> global id (-1: empty), first arena record, length
  int global_of(int s) const { return slot_[s].global; }
  long long off_of(int s) const { return slot_[s].off; }
  int len_of(int s) const { return slot_[s].global < 0 ? 0 : slot_[s].len; }
  int slot_of(int global) const {
    auto it = where_.find(global);
    return it == where_.end() ? -1 : it->second;
  }

  // Makes the n targets ids[] (ids into a store of n_store targets with lengths L and first records src_off) resident.
  // local[n] receives their slots; items the copies the caller must make; freed the slots that lost their target and
  // got no new one.  Returns 0, or -1 (an id outside the store: *bad = its position) or -2 (the distinct targets need
  // *need_slots slots / *need_cols columns, more than the shard has); after a failure nothing has changed.
  int request(int n, const int32_t* ids, int n_store, const int32_t* L, const long long* src_off, int32_t* local,
              std::vector<StageItem>* items, std::vector<int>* freed, StageStats* st, int* bad, long long* need_slots,
              long long* need_cols) {
    items->clear();
    freed->clear();
    *st = StageStats{0, 0, 0, 0};
    std::vector<int> uniq;
    {
      std::unordered_map<int, int> seen;
      long long cols = 0;
      for (int k = 0; k < n; ++k) {
        if (ids[k] < 0 || ids[k] >= n_store) { *bad = k; return -1; }
        if (seen.emplace(ids[k], 1).second) { uniq.push_back(ids[k]); cols += L[ids[k]]; }
      }
      *need_slots = (long long)uniq.size();
      *need_cols = cols;
      if ((long long)uniq.size() > (long long)slot_.size() || cols > cap_cols_) return -2;
    }
    ++stamp_;
    std::vector<int> missing;
    for (int g : uniq) {
      const int s = slot_of(g);
      if (s < 0) { missing.push_back(g); continue; }
      touch(s);
    }
    std::set<int> was_freed;
    for (int g : missing) {
      const int len = L[g];
      if (free_slots_.empty()) evict_lru(&was_freed, st);
      long long off = take_run(len);
      while (off < 0 && !lru_.empty() && lru_.begin()->first != stamp_) {
        evict_lru(&was_freed, st);
        off = take_run(len);
      }
      if (off < 0) {           // only this request's targets are left and they fragment the arena: lay them out again
        repack(items, src_off);
        off = take_run(len);
      }
      const int s = free_slots_.back();
      free_slots_.pop_back();
      was_freed.erase(s);
      slot_[s] = Slot{g, off, len, stamp_};
      lru_.insert({stamp_, s});
      where_[g] = s;
      items->push_back(StageItem{src_off[g], off, len, s, g});
    }
    for (int k = 0; k < n; ++k) local[k] = where_[ids[k]];
    freed->assign(was_freed.begin(), was_freed.end());
    st->copied = (long long)items->size();
    st->hits = (long long)uniq.size() - st->copied;
    for (const StageItem& it : *items) st->bytes += (long long)it.len * 112 + 80 + 12;   // records, pav, L and col_off
    return 0;
  }

 private:
  struct Slot {
    int global = -1;
    long long off = 0;
    int len = 0;
    unsigned long long used = 0;
  };

  void touch(int s) {
    lru_.erase({slot_[s].used, s});
    slot_[s].used = stamp_;
    lru_.insert({stamp_, s});
  }
  // first free run of at least len records, or -1
  long long take_run(int len) {
    for (auto it = free_.begin(); it != free_.end(); ++it) {
      if (it->second < len) continue;
      const long long off = it->first, rest = it->second - len;
      free_.erase(it);
      if (rest > 0) free_[off + len] = rest;
      return off;
    }
    return -1;
  }
  void give_run(long long off, long long len) {
    auto nx = free_.lower_bound(off);
    if (nx != free_.begin()) {
      auto pv = std::prev(nx);
      if (pv->first + pv->second == off) { off = pv->first; len += pv->second; free_.erase(pv); }
    }
    if (nx != free_.end() && off + len == nx->first) { len += nx->second; free_.erase(nx); }
    free_[off] = len;
  }
  // evicts the least recently staged target that the current request does not name (the caller has checked that the
  // request fits, so there is one whenever a slot is needed)
  void evict_lru(std::set<int>* was_freed, StageStats* st) {
    const int s = lru_.begin()->second;
    lru_.erase(lru_.begin());
    where_.erase(slot_[s].global);
    give_run(slot_[s].off, slot_[s].len);
    slot_[s].global = -1;
    free_slots_.push_back(s);
    was_freed->insert(s);
    st->evicted++;
  }
  // every resident target belongs to the current request: give each a run from column 0 on and copy all of them again
  void repack(std::vector<StageItem>* items, const long long* src_off) {
    items->clear();
    free_.clear();
    long long at = 0;
    for (const auto& us : lru_) {
      Slot& sl = slot_[us.second];
      sl.off = at;
      at += sl.len;
      items->push_back(StageItem{src_off[sl.global], sl.off, sl.len, us.second, sl.global});
    }
    if (at < cap_cols_) free_[at] = cap_cols_ - at;
  }

  long long cap_cols_;
  unsigned long long stamp_ = 0;
  std::vector<Slot> slot_;
  std::vector<int> free_slots_;
  std::map<long long, long long> free_;                  // free arena runs: first record -> length
  std::set<std::pair<unsigned long long, int>> lru_;     // (stamp of the last request that named it, slot)
  std::unordered_map<int, int> where_;                   // global id -> slot
};

}  // namespace hhg
