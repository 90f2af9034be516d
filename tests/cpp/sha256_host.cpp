// Host execution of the DEVICE SHA-256 in plonky3_b200/csrc/hash_core.cuh, compiled as plain C++.  A filter over input lines:
//   <hex message>           ("-" for the empty message): its 32-byte SHA-256 digest in hex
//   c <64 hex state> <128 hex block>
//                           one raw compression (compress256) of the 64-byte block from the given 32-byte state, both as
//                           big-endian words: the new state in hex
// tests/test_sha256_config_cpu.py compares them with hashlib, the reference's own test vectors and tests/sha256_air_oracle.py.
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <iostream>
#include <string>
#include <vector>
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned shift) {
    return (unsigned)(((((unsigned long long)hi << 32) | lo) << (shift & 31)) >> 32);
}
#include "../../plonky3_b200/csrc/hash_core.cuh"

static std::vector<unsigned char> unhex(const std::string &s) {
    std::vector<unsigned char> b(s.size() / 2);
    for (size_t i = 0; i < b.size(); i++) b[i] = (unsigned char)std::stoul(s.substr(2 * i, 2), nullptr, 16);
    return b;
}
static p3::u32 be(const unsigned char *p) { return (p3::u32)p[0] << 24 | (p3::u32)p[1] << 16 | (p3::u32)p[2] << 8 | p[3]; }

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        if (line.rfind("c ", 0) == 0) {
            const size_t sp = line.find(' ', 2);
            if (sp == std::string::npos) return 2;
            const auto st = unhex(line.substr(2, sp - 2)), blk = unhex(line.substr(sp + 1));
            if (st.size() != 32 || blk.size() != 64) return 2;
            p3::u32 s[8], w[16];
            for (int i = 0; i < 8; i++) s[i] = be(&st[4 * i]);
            for (int i = 0; i < 16; i++) w[i] = be(&blk[4 * i]);
            p3::sha256_compress(s, w);
            for (p3::u32 v : s) printf("%08x", v);
            printf("\n");
            continue;
        }
        if (line == "-") line.clear();
        if (line.size() % 2) return 2;
        const auto msg = unhex(line);
        unsigned char out[32];
        p3::sha256(msg.data(), msg.size(), out);
        for (unsigned char c : out) printf("%02x", c);
        printf("\n");
    }
    return 0;
}
