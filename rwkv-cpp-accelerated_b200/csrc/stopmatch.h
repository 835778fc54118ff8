// stopmatch.h — stop strings (include/rwkv_b200.h, rwkv_b200_stop_set_add): the byte automaton of a stop set and the
// walk of one token's bytes through it. Plain C++ apart from the qualifiers, so the host builds the automaton, the
// decoding kernels walk it, and a host test compiles both with g++.
//
// The automaton is the Aho–Corasick DFA of the set's strings s_0 .. s_(n-1), dense: next[q * 256 + c] and hit[q], u32.
// State q stands for a prefix of some string: the q-th distinct prefix in order of first appearance (state 0 the empty
// prefix, then the prefixes of s_0 by length, then those of s_1 that are new, and so on), so a host can restate it.
// Reading byte c in state q goes to the longest suffix of (prefix q) + c that is a prefix of some string, and hit[q] =
// 1 + the lowest i such that s_i is a suffix of prefix q, or 0. After any bytes B from state 0, the state is the
// longest suffix of B that is a prefix of some string, and hit != 0 exactly when some string ends at B's last byte.
#pragma once
#include <cstdint>
#include <vector>

#ifdef __CUDACC__
#define STOPMATCH_HD __host__ __device__
#else
#define STOPMATCH_HD
#endif

namespace stopmatch {

constexpr uint32_t kNone = 0xFFFFFFFFu;

// The automaton of the strings bytes[start[i] .. start[i + 1]), i < n (each non-empty; the caller checks). Returns the
// number of states; next gets [states][256], hit [states].
inline uint32_t build(const unsigned long long *start, const unsigned char *bytes, unsigned long long n,
                      std::vector<uint32_t> &next, std::vector<uint32_t> &hit) {
    next.assign(256, kNone);
    hit.assign(1, 0);
    // the trie, states numbered in order of first appearance
    for (unsigned long long i = 0; i < n; ++i) {
        uint32_t q = 0;
        for (unsigned long long k = start[i]; k < start[i + 1]; ++k) {
            uint32_t &t = next[(size_t)q * 256 + bytes[k]];
            if (t == kNone) {
                t = (uint32_t)hit.size();
                hit.push_back(0);
                next.resize(next.size() + 256, kNone);
            }
            q = next[(size_t)q * 256 + bytes[k]];
        }
        if (hit[q] == 0) hit[q] = (uint32_t)(i + 1); // a duplicate keeps the lower index
    }
    // failure links in breadth-first order: a state's shorter suffixes are complete before it
    const uint32_t states = (uint32_t)hit.size();
    std::vector<uint32_t> fail(states, 0), order;
    order.reserve(states);
    for (int c = 0; c < 256; ++c) {
        uint32_t &t = next[c];
        if (t == kNone) t = 0;
        else order.push_back(t);
    }
    for (size_t h = 0; h < order.size(); ++h) {
        const uint32_t q = order[h], f = fail[q];
        if (hit[f] && (hit[q] == 0 || hit[f] < hit[q])) hit[q] = hit[f];
        for (int c = 0; c < 256; ++c) {
            uint32_t &t = next[(size_t)q * 256 + c];
            const uint32_t via = next[(size_t)f * 256 + c];
            if (t == kNone) {
                t = via;
            } else {
                fail[t] = via;
                order.push_back(t);
            }
        }
    }
    return states;
}

// Walk bytes b[0 .. n) from state q, stopping at the first byte whose state has a hit. Returns that hit (0: none);
// q becomes the state after the last byte walked and tail the bytes of b after it.
STOPMATCH_HD inline uint32_t walk(const uint32_t *next, const uint32_t *hit, uint32_t &q, const unsigned char *b,
                                  unsigned long long n, unsigned long long &tail) {
    uint32_t s = q;
    for (unsigned long long i = 0; i < n; ++i) {
        s = next[(size_t)s * 256 + b[i]];
        const uint32_t h = hit[s];
        if (h) {
            q = s;
            tail = n - i - 1;
            return h;
        }
    }
    q = s;
    tail = 0;
    return 0;
}

} // namespace stopmatch
