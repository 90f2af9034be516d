// Host execution of the DEVICE Keccak-256 in plonky3_b200/csrc/hash_core.cuh, compiled as plain C++.  A filter: every input line is
// a message in hex ("-" for the empty message); every output line is its 32-byte digest in hex.  tests/test_keccak_transcript_cpu.py
// compares them with the published vectors and with a Python restatement over the oracle's Keccak-f.
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

int main() {
    std::string line;
    while (std::getline(std::cin, line)) {
        if (line == "-") line.clear();
        if (line.size() % 2) return 2;
        std::vector<unsigned char> msg(line.size() / 2);
        for (size_t i = 0; i < msg.size(); i++) msg[i] = (unsigned char)std::stoul(line.substr(2 * i, 2), nullptr, 16);
        unsigned char out[32];
        p3::keccak256(msg.data(), msg.size(), out);
        for (unsigned char c : out) printf("%02x", c);
        printf("\n");
    }
    return 0;
}
