// prefix_index.h — host-only index of a prefix state cache (include/rwkv_b200.h, "Prefix state cache"). No CUDA here,
// so tests/helpers/prefix_index_test.cpp drives it on the CPU.
//
// An entry holds the recurrent state (xy, aa, bb, dd) after a token sequence run from the zero state. Its key is the
// pair (adapter binding, exact token sequence). The index only decides which entry a snapshot or a restore uses; the
// device copies live in the cache's pool (prefix.cuh) and move on the model's one stream, in the order the host enqueues
// them. So a restore enqueued before a pass that overwrites its entry reads the old contents, and a lookup sees every
// entry whose snapshot pass has already been enqueued.
//
// Policy:
//  - lookup: the longest live entry whose key is a prefix of the tokens under the same binding. Keys are compared token
//    by token; the hash only finds candidates, so a collision can cost time but never returns a wrong entry;
//  - snapshot: a key that already exists is not written again and counts as a use of its entry. Otherwise a free entry,
//    else the least recently used evictable entry, is taken. Evictable: live, not pinned, and no live entry under the
//    same binding extends its key (leaves first). With none, the snapshot is skipped and counted;
//  - every use (a hit, an existing key, a new snapshot, an insert) stamps the entry with the next value of a counter, so
//    the order, and every count, is a function of the calls alone;
//  - entries taken for the layout being built are pinned until unpin_all(), so a layout never evicts its own snapshots.
#pragma once

#include <algorithm>
#include <cstdint>
#include <unordered_map>
#include <vector>

namespace prefix {

struct Stats {
    unsigned long long live = 0, lookups = 0, hit_tokens = 0, prefilled_tokens = 0, snapshots = 0, skipped = 0, evictions = 0;
};

class Index {
  public:
    // hash_mask: the bits of the hash the buckets use (tests force collisions with a small mask)
    explicit Index(size_t capacity, uint64_t hash_mask = ~0ull) : ent_(capacity), mask_(hash_mask) {}

    size_t capacity() const { return ent_.size(); }
    const Stats &stats() const { return st_; }
    Stats &stats() { return st_; }

    // The entry whose key is exactly (binding, tokens[0 .. n)), or -1.
    long find(unsigned long long binding, const unsigned long long *tokens, size_t n) const {
        uint64_t h = seed(binding);
        for (size_t i = 0; i < n; ++i) h = mix(h, tokens[i]);
        return match(h, binding, tokens, n);
    }

    // The longest live entry whose key is a prefix of tokens[0 .. limit) under `binding`: returns its length (0: none)
    // and the entry in *entry (-1: none). A hit is a use of the entry. Counts one lookup and the hit tokens.
    size_t lookup(unsigned long long binding, const unsigned long long *tokens, size_t limit, long *entry) {
        st_.lookups += 1;
        *entry = -1;
        std::vector<uint64_t> h;
        hashes(binding, tokens, limit, h);
        for (size_t n = limit; n >= 1; --n) {
            const long e = match(h[n], binding, tokens, n);
            if (e >= 0) {
                touch(e);
                *entry = e;
                st_.hit_tokens += n;
                return n;
            }
        }
        return 0;
    }

    // An entry for the state after (binding, tokens[0 .. n)), n >= 1, pinned. *fresh = true: the caller must write it
    // (a snapshot taken); false: the key exists and the entry is returned as is (a use). Returns -1 when every entry is
    // pinned or extended by a pinned entry (the snapshot is skipped and counted).
    long take(unsigned long long binding, const unsigned long long *tokens, size_t n, bool *fresh) {
        std::vector<uint64_t> h;
        hashes(binding, tokens, n, h);
        long e = match(h[n], binding, tokens, n);
        *fresh = e < 0;
        if (e >= 0) {
            touch(e);
            pin(e);
            return e;
        }
        e = free_entry();
        if (e < 0) {
            st_.skipped += 1;
            return -1;
        }
        Entry &x = ent_[(size_t)e];
        x.live = true;
        x.binding = binding;
        x.key.assign(tokens, tokens + n);
        x.ext = 0;
        for (const Entry &y : ent_) // live entries that extend this key (an insert, or a key a lookup limit skipped)
            if (y.live && &y != &x && y.binding == binding && y.key.size() > n && std::equal(tokens, tokens + n, y.key.begin()))
                x.ext += 1;
        buckets_.emplace(h[n] & mask_, e);
        for (size_t k = 1; k < n; ++k) // the live entries this key extends
            if (long f = match(h[k], binding, tokens, k); f >= 0) ent_[(size_t)f].ext += 1;
        st_.live += 1;
        st_.snapshots += 1;
        touch(e);
        pin(e);
        return e;
    }

    void unpin_all() {
        for (long e : pinned_) ent_[(size_t)e].pinned = false;
        pinned_.clear();
    }

    // Forget every entry; the counters other than `live` keep counting.
    void clear() {
        for (Entry &x : ent_) x = Entry{};
        buckets_.clear();
        pinned_.clear();
        st_.live = 0;
    }

    // For tests: the key of a live entry (empty when free).
    const std::vector<unsigned long long> &key(long e) const { return ent_[(size_t)e].key; }
    bool live(long e) const { return ent_[(size_t)e].live; }

  private:
    struct Entry {
        bool live = false, pinned = false;
        unsigned long long binding = 0;
        std::vector<unsigned long long> key;
        unsigned long long used = 0; // counter value of the last use
        unsigned long long ext = 0;  // live entries under the same binding whose key extends this one
    };

    static uint64_t mix(uint64_t h, uint64_t x) { // splitmix64 of h ^ x
        uint64_t z = h ^ (x + 0x9e3779b97f4a7c15ull);
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        return z ^ (z >> 31);
    }
    static uint64_t seed(unsigned long long binding) { return mix(0x243f6a8885a308d3ull, binding); }
    // h[k] = hash of (binding, tokens[0 .. k)) for k = 0..n
    static void hashes(unsigned long long binding, const unsigned long long *tokens, size_t n, std::vector<uint64_t> &h) {
        h.resize(n + 1);
        h[0] = seed(binding);
        for (size_t i = 0; i < n; ++i) h[i + 1] = mix(h[i], tokens[i]);
    }
    // Every candidate of the bucket is compared by its binding and tokens: equal hashes never decide a match.
    long match(uint64_t h, unsigned long long binding, const unsigned long long *tokens, size_t n) const {
        auto r = buckets_.equal_range(h & mask_);
        for (auto it = r.first; it != r.second; ++it) {
            const Entry &x = ent_[(size_t)it->second];
            if (x.binding == binding && x.key.size() == n && std::equal(x.key.begin(), x.key.end(), tokens)) return it->second;
        }
        return -1;
    }
    void touch(long e) { ent_[(size_t)e].used = ++clock_; }
    void pin(long e) {
        if (!ent_[(size_t)e].pinned) pinned_.push_back(e);
        ent_[(size_t)e].pinned = true;
    }
    // A free entry (the lowest index), else the least recently used evictable one, evicted; -1 when there is none.
    long free_entry() {
        long best = -1;
        for (size_t i = 0; i < ent_.size(); ++i) {
            const Entry &x = ent_[i];
            if (!x.live) return (long)i;
            if (!x.pinned && x.ext == 0 && (best < 0 || x.used < ent_[(size_t)best].used)) best = (long)i;
        }
        if (best >= 0) evict(best);
        return best;
    }
    void evict(long e) {
        Entry &x = ent_[(size_t)e];
        std::vector<uint64_t> h;
        hashes(x.binding, x.key.data(), x.key.size(), h);
        for (size_t k = 1; k < x.key.size(); ++k)
            if (long f = match(h[k], x.binding, x.key.data(), k); f >= 0) ent_[(size_t)f].ext -= 1;
        auto r = buckets_.equal_range(h.back() & mask_);
        for (auto it = r.first; it != r.second; ++it)
            if (it->second == e) {
                buckets_.erase(it);
                break;
            }
        x = Entry{};
        st_.live -= 1;
        st_.evictions += 1;
    }

    std::vector<Entry> ent_;
    std::unordered_multimap<uint64_t, long> buckets_;
    std::vector<long> pinned_;
    uint64_t mask_;
    unsigned long long clock_ = 0;
    Stats st_;
};

} // namespace prefix
