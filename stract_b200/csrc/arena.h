// arena.h -- host-side sub-allocator over a few large device slabs (opt-in: SB200_ARENA=1).
//
// Why: one sb200_graph_create at C2 size allocates and frees tens of GB of staging temporaries.  cudaMalloc/cudaFree
// of such sizes are slow, and the driver's stream-ordered pool (cudaMallocAsync), which replaced them, still stalls
// when it has to grow or re-map.  A create performs the same allocation sequence every time, so a
// deterministic best-fit allocator over slabs that are never returned reaches a steady state after the first
// create and costs no driver call afterwards.
//
// Ordering contract (the same one cudaFreeAsync(p, stream) gives): a block is freed "on" a stream, meaning all
// work that touches it has been enqueued on (or joined into) that stream.  A later allocation for the SAME stream
// may reuse the block at once -- its first use is enqueued behind the old users.  A different stream first
// synchronises the old one (rare: one handle = one stream; handles retire their stream when destroyed).
//
// Pure host logic over an abstract backend, so tests/test_arena_host.py exercises it on the CPU with malloc.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <iterator>
#include <map>
#include <mutex>
#include <unordered_map>
#include <vector>

namespace sb200 {

struct ArenaBackend {
  void* (*slab_alloc)(size_t bytes);         // nullptr on failure
  void (*slab_free)(void* p);
  void (*stream_sync)(void* stream);         // block the host until `stream` is idle
};

class Arena {
 public:
  static constexpr size_t ALIGN = 512;
  explicit Arena(ArenaBackend be, size_t min_slab_bytes = (size_t)2 << 30) : be_(be), min_slab_(min_slab_bytes) {}
  ~Arena() { for (auto& s : slabs_) be_.slab_free(s.raw); }
  Arena(const Arena&) = delete;
  Arena& operator=(const Arena&) = delete;

  void* alloc(size_t bytes, void* stream) {
    if (bytes == 0) bytes = 1;
    bytes = (bytes + ALIGN - 1) / ALIGN * ALIGN;
    std::lock_guard<std::mutex> lk(mu_);
    for (int attempt = 0; attempt < 2; attempt++) {
      // best fit: the smallest free block that holds `bytes`; ties -> lowest slab, lowest offset (deterministic)
      int bs = -1; size_t boff = 0, blen = ~(size_t)0;
      for (size_t si = 0; si < slabs_.size(); si++)
        for (auto& kv : slabs_[si].free_blocks)
          if (kv.second.len >= bytes && kv.second.len < blen) { bs = (int)si; boff = kv.first; blen = kv.second.len; }
      if (bs >= 0) {
        Slab& s = slabs_[bs];
        void* tag = s.free_blocks[boff].tag;
        s.free_blocks.erase(boff);
        if (blen > bytes) s.free_blocks[boff + bytes] = Block{blen - bytes, tag};
        if (tag && tag != stream) { be_.stream_sync(tag); clear_tag_locked(tag); }
        void* p = s.base + boff;
        live_[p] = Live{bs, bytes};
        in_use_ += bytes;
        if (in_use_ > peak_) peak_ = in_use_;
        return p;
      }
      if (attempt == 1) break;
      size_t want = bytes > min_slab_ ? bytes : min_slab_;
      want = (want + ALIGN + ((size_t)2 << 20) - 1) / ((size_t)2 << 20) * ((size_t)2 << 20);
      char* base = (char*)be_.slab_alloc(want);
      if (!base && want > bytes + ALIGN) {  // not enough memory for a roomy slab: try an exact one
        want = (bytes + ALIGN + ((size_t)2 << 20) - 1) / ((size_t)2 << 20) * ((size_t)2 << 20);
        base = (char*)be_.slab_alloc(want);
      }
      if (!base) return nullptr;
      // the backend's base need not be ALIGN-aligned (cudaMalloc: 256 B, malloc: 16 B): carve the aligned interior
      const size_t pad = (ALIGN - (size_t)((uintptr_t)base % ALIGN)) % ALIGN;
      const size_t usable = (want - pad) / ALIGN * ALIGN;
      if (usable < bytes) { be_.slab_free(base); return nullptr; }
      Slab s; s.raw = base; s.base = base + pad; s.size = usable; s.reserved = want; s.free_blocks[0] = Block{usable, nullptr};
      slabs_.push_back(std::move(s));
      reserved_ += want;
    }
    return nullptr;
  }

  // false: `p` did not come from this arena
  bool free(void* p, void* stream) {
    std::lock_guard<std::mutex> lk(mu_);
    auto it = live_.find(p);
    if (it == live_.end()) return false;
    const Live l = it->second;
    live_.erase(it);
    in_use_ -= l.len;
    Slab& s = slabs_[l.slab];
    insert_free_locked(s, (size_t)((char*)p - s.base), l.len, stream);
    return true;
  }

  // the stream is idle and about to be destroyed: its blocks become reusable by anyone
  void retire_stream(void* stream) {
    if (!stream) return;
    std::lock_guard<std::mutex> lk(mu_);
    clear_tag_locked(stream);
  }

  // give slabs without live allocations back to the backend
  void trim() {
    std::lock_guard<std::mutex> lk(mu_);
    std::vector<Slab> keep;
    std::vector<int> remap(slabs_.size(), -1);
    for (size_t si = 0; si < slabs_.size(); si++) {
      Slab& s = slabs_[si];
      size_t free_len = 0;
      for (auto& kv : s.free_blocks) free_len += kv.second.len;
      if (free_len == s.size) {  // nothing live in it (free neighbours with different stream tags stay unmerged)
        for (auto& kv : s.free_blocks) if (kv.second.tag) be_.stream_sync(kv.second.tag);
        be_.slab_free(s.raw); reserved_ -= s.reserved;
      } else { remap[si] = (int)keep.size(); keep.push_back(std::move(s)); }
    }
    slabs_.swap(keep);
    for (auto& kv : live_) kv.second.slab = remap[kv.second.slab];
  }

  size_t reserved() const { return reserved_; }
  size_t in_use() const { return in_use_; }
  size_t peak() const { return peak_; }
  size_t n_slabs() const { return slabs_.size(); }
  size_t n_free_blocks() const { size_t n = 0; for (auto& s : slabs_) n += s.free_blocks.size(); return n; }
  size_t n_live() const { return live_.size(); }

  // consistency check for the self-test: blocks tile every slab exactly, nothing overlaps, neighbours that could
  // have been merged were merged
  bool check() const {
    for (size_t si = 0; si < slabs_.size(); si++) {
      const Slab& s = slabs_[si];
      std::map<size_t, size_t> all;  // off -> len
      for (auto& kv : s.free_blocks) all[kv.first] = kv.second.len;
      for (auto& kv : live_) if (kv.second.slab == (int)si) all[(size_t)((char*)kv.first - s.base)] = kv.second.len;
      size_t pos = 0;
      for (auto& kv : all) { if (kv.first != pos || kv.second == 0 || kv.first % ALIGN) return false; pos += kv.second; }
      if (pos != s.size) return false;
      const Block* prev = nullptr; size_t prev_end = 0;
      for (auto& kv : s.free_blocks) {
        if (prev && prev_end == kv.first && prev->tag == kv.second.tag) return false;  // unmerged neighbours
        prev = &kv.second; prev_end = kv.first + kv.second.len;
      }
    }
    return true;
  }

 private:
  struct Block { size_t len; void* tag; };
  struct Slab { char* raw = nullptr; char* base = nullptr; size_t size = 0, reserved = 0; std::map<size_t, Block> free_blocks; };
  struct Live { int slab; size_t len; };

  void insert_free_locked(Slab& s, size_t off, size_t len, void* tag) {
    auto nx = s.free_blocks.lower_bound(off);
    if (nx != s.free_blocks.end() && off + len == nx->first && nx->second.tag == tag) { len += nx->second.len; nx = s.free_blocks.erase(nx); }
    if (nx != s.free_blocks.begin()) {
      auto pv = std::prev(nx);
      if (pv->first + pv->second.len == off && pv->second.tag == tag) { pv->second.len += len; return; }
    }
    s.free_blocks[off] = Block{len, tag};
  }
  void clear_tag_locked(void* tag) {
    for (auto& s : slabs_) {
      bool any = false;
      for (auto& kv : s.free_blocks) if (kv.second.tag == tag) { kv.second.tag = nullptr; any = true; }
      if (!any) continue;
      std::map<size_t, Block> merged;  // untagged neighbours may now touch: rebuild with merging
      for (auto& kv : s.free_blocks) {
        if (!merged.empty()) {
          auto& last = *merged.rbegin();
          if (last.first + last.second.len == kv.first && last.second.tag == kv.second.tag) { last.second.len += kv.second.len; continue; }
        }
        merged[kv.first] = kv.second;
      }
      s.free_blocks.swap(merged);
    }
  }

  ArenaBackend be_;
  size_t min_slab_;
  std::vector<Slab> slabs_;
  std::unordered_map<void*, Live> live_;
  size_t reserved_ = 0, in_use_ = 0, peak_ = 0;
  mutable std::mutex mu_;
};

}  // namespace sb200
