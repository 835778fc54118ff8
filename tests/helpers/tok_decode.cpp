// tok_decode.cpp — one token id per input line -> the hex of GPT2Tokenizer::decode({id}) of this repository's
// include/rwkv/tokenizer/tokenizer.h, one line each.
#include <cstdio>
#include <iostream>
#include <string>
#include "rwkv/tokenizer/tokenizer.h"

int main(int argc, char **argv) {
    if (argc < 3) return 1;
    auto t = GPT2Tokenizer::load(argv[1], argv[2]);
    if (!t.has_value()) return 2;
    GPT2Tokenizer tok = t.value();
    std::string line;
    while (std::getline(std::cin, line)) {
        const std::string back = tok.decode({std::stoll(line)});
        for (unsigned char c : back) printf("%02x", c);
        printf("\n");
    }
    return 0;
}
