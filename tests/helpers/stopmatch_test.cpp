// Host driver of csrc/stopmatch.h for tests/test_stop_host.py. Reads from stdin, whitespace separated, byte strings in
// hex ("-" for an empty one):
//   n_strings  string_0 .. string_(n-1)  print_table(0/1)  start_state  n_chunks  chunk_0 .. chunk_(m-1)
// Prints the number of states; with print_table, per state its hit and its 256 next states on one line; then per
// chunk "hit state tail" after stopmatch::walk from the previous chunk's state.
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>

#include "../../rwkv-cpp-accelerated_b200/csrc/stopmatch.h"

static std::vector<unsigned char> unhex(const std::string &s) {
    std::vector<unsigned char> out;
    if (s == "-") return out;
    for (size_t i = 0; i + 1 < s.size(); i += 2) out.push_back((unsigned char)std::stoul(s.substr(i, 2), nullptr, 16));
    return out;
}

int main() {
    unsigned long long n = 0;
    std::cin >> n;
    std::vector<unsigned long long> start{0};
    std::vector<unsigned char> bytes;
    for (unsigned long long i = 0; i < n; ++i) {
        std::string h;
        std::cin >> h;
        const std::vector<unsigned char> b = unhex(h);
        bytes.insert(bytes.end(), b.begin(), b.end());
        start.push_back(bytes.size());
    }
    int table = 0;
    unsigned long long q0 = 0, m = 0;
    std::cin >> table >> q0 >> m;
    std::vector<uint32_t> next, hit;
    const uint32_t states = stopmatch::build(start.data(), bytes.data(), n, next, hit);
    printf("%u\n", states);
    for (uint32_t q = 0; table && q < states; ++q) {
        printf("%u", hit[q]);
        for (int c = 0; c < 256; ++c) printf(" %u", next[(size_t)q * 256 + c]);
        printf("\n");
    }
    uint32_t q = (uint32_t)q0;
    for (unsigned long long j = 0; j < m; ++j) {
        std::string h;
        std::cin >> h;
        const std::vector<unsigned char> b = unhex(h);
        unsigned long long tail = 0;
        const uint32_t got = stopmatch::walk(next.data(), hit.data(), q, b.data(), b.size(), tail);
        printf("%u %u %llu\n", got, q, tail);
    }
    return 0;
}
