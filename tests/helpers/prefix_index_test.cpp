// Host driver of csrc/prefix_index.h for tests/test_prefix_host.py. Reads commands from stdin, one per line; a token
// list is its length followed by the tokens:
//   new capacity hash_mask            a fresh index (hash_mask 0 puts every key in one bucket)
//   lookup binding limit tokens       prints "length entry" of the longest live prefix of tokens[0 .. limit)
//   take binding tokens               prints "entry fresh" (entry -1: skipped)
//   find binding tokens               prints the entry or -1
//   unpin | clear
//   stats                             prints live lookups hit_tokens prefilled_tokens snapshots skipped evictions
#include <cstdio>
#include <iostream>
#include <memory>
#include <string>
#include <vector>

#include "../../rwkv-cpp-accelerated_b200/csrc/prefix_index.h"

static std::vector<unsigned long long> read_tokens() {
    size_t n = 0;
    std::cin >> n;
    std::vector<unsigned long long> t(n);
    for (auto &x : t) std::cin >> x;
    return t;
}

int main() {
    std::unique_ptr<prefix::Index> ix;
    std::string cmd;
    while (std::cin >> cmd) {
        if (cmd == "new") {
            size_t cap = 0;
            unsigned long long mask = 0;
            std::cin >> cap >> mask;
            ix.reset(new prefix::Index(cap, mask));
        } else if (cmd == "lookup") {
            unsigned long long b = 0, limit = 0;
            std::cin >> b >> limit;
            const std::vector<unsigned long long> t = read_tokens();
            long e = -1;
            const size_t r = ix->lookup(b, t.data(), limit, &e);
            printf("%zu %ld\n", r, e);
        } else if (cmd == "take") {
            unsigned long long b = 0;
            std::cin >> b;
            const std::vector<unsigned long long> t = read_tokens();
            bool fresh = false;
            const long e = ix->take(b, t.data(), t.size(), &fresh);
            printf("%ld %d\n", e, e >= 0 && fresh ? 1 : 0);
        } else if (cmd == "find") {
            unsigned long long b = 0;
            std::cin >> b;
            const std::vector<unsigned long long> t = read_tokens();
            printf("%ld\n", ix->find(b, t.data(), t.size()));
        } else if (cmd == "unpin") {
            ix->unpin_all();
        } else if (cmd == "clear") {
            ix->clear();
        } else if (cmd == "stats") {
            const prefix::Stats &s = ix->stats();
            printf("%llu %llu %llu %llu %llu %llu %llu\n", s.live, s.lookups, s.hit_tokens, s.prefilled_tokens, s.snapshots,
                   s.skipped, s.evictions);
        }
    }
    return 0;
}
