// Host execution of the DEVICE byte transcript (SerializingChallenger32 over Keccak-256 or SHA-256) in
// plonky3_b200/csrc/hash_core.cuh, compiled as plain C++: the state machine the observe, sample and grind kernels of challenger.cu
// run, on a host state array.  A filter over input lines; every command answers one line, so a caller can drive it step by step:
//   new <k|s> <field> [<word> ...]   a transcript over Keccak-256 (k) or SHA-256 (s) and field 0 (BabyBear) / 1 (KoalaBear), the
//                                    words observed as their own bytes (from_hasher's initial state): its handle
//   <h> obs <word> ...               observe Montgomery words: "ok"
//   <h> dig <word> ...               observe words as their own bytes (digests): "ok"
//   <h> sample <n>                   n field elements, as Montgomery words
//   <h> bits <bits>                  sample_bits(bits)
//   <h> clone                        a copy of the transcript: its handle
//   <h> wit <bits> <c>               1 if the canonical value c is a witness for `bits` (the grind kernel's test), else 0
//   <h> grind <bits>                 the smallest witness by a sequential search with the same test, observed and checked like
//                                    check_witness: the witness as a Montgomery word
// Words are decimal.  tests/test_transcript_host_cpu.py compares the answers with the restatements in tests/keccak_transcript.py
// and tests/sha256_config.py.
#include <cstdint>
#include <cstdio>
#include <iostream>
#include <sstream>
#include <string>
#include <type_traits>
#include <vector>
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned shift) {
    return (unsigned)(((((unsigned long long)hi << 32) | lo) << (shift & 31)) >> 32);
}
#include "../../plonky3_b200/csrc/hash_core.cuh"

using p3::u32;

struct Transcript {
    bool sha256;
    int field;
    std::vector<u32> st;
};

// fn(policy, field) with both as types, like challenger.cu's dispatcher
template <class Fn> static void dispatch(const Transcript &t, Fn &&fn) {
    auto by_field = [&](auto h) {
        if (t.field == p3::BABY_BEAR) fn(h, std::integral_constant<int, p3::BABY_BEAR>());
        else fn(h, std::integral_constant<int, p3::KOALA_BEAR>());
    };
    if (t.sha256) by_field(p3::Sha256Policy());
    else by_field(p3::Keccak256Policy());
}

static std::vector<u32> read_words(std::istringstream &in) {
    std::vector<u32> v;
    unsigned long long x;
    while (in >> x) v.push_back((u32)x);
    return v;
}

int main() {
    std::vector<Transcript> ts;
    std::string line;
    while (std::getline(std::cin, line)) {
        std::istringstream in(line);
        std::string head, cmd;
        in >> head;
        if (head == "new") {
            std::string hash;
            Transcript t;
            in >> hash >> t.field;
            if ((hash != "k" && hash != "s") || (t.field != p3::BABY_BEAR && t.field != p3::KOALA_BEAR)) return 2;
            t.sha256 = hash == "s";
            t.st.assign(p3::TR_WORDS, 0);
            const std::vector<u32> init = read_words(in);
            dispatch(t, [&](auto h, auto f) {
                using H = decltype(h);
                H::init(t.st.data());
                p3::transcript_observe<H, decltype(f)::value, false>(t.st.data(), init.data(), init.size());
            });
            ts.push_back(t);
            printf("%zu\n", ts.size() - 1);
            fflush(stdout);
            continue;
        }
        const size_t i = std::stoul(head);
        if (i >= ts.size()) return 2;
        in >> cmd;
        if (cmd == "clone") {
            ts.push_back(ts[i]);
            printf("%zu\n", ts.size() - 1);
            fflush(stdout);
            continue;
        }
        Transcript &t = ts[i];
        u32 *st = t.st.data();
        bool ok = true;
        dispatch(t, [&](auto h, auto f) {
            using H = decltype(h);
            constexpr int F = decltype(f)::value;
            if (cmd == "obs" || cmd == "dig") {
                const std::vector<u32> v = read_words(in);
                if (cmd == "obs") p3::transcript_observe<H, F, true>(st, v.data(), v.size());
                else p3::transcript_observe<H, F, false>(st, v.data(), v.size());
                printf("ok\n");
            } else if (cmd == "sample") {
                size_t n = 0;
                in >> n;
                std::vector<u32> out(n);
                p3::transcript_sample<H, F>(st, out.data(), n, false, 0);
                for (size_t j = 0; j < n; j++) printf(j ? " %u" : "%u", out[j]);
                printf("\n");
            } else if (cmd == "bits") {
                unsigned bits = 0;
                in >> bits;
                u32 s;
                p3::transcript_sample<H, F>(st, &s, 1, true, (1u << bits) - 1u);
                printf("%u\n", s);
            } else if (cmd == "wit") {
                unsigned bits = 0;
                u32 c = 0;
                in >> bits >> c;
                printf("%d\n", p3::transcript_is_witness<H>(st, c, (1u << bits) - 1u) ? 1 : 0);
            } else if (cmd == "grind") {
                unsigned bits = 0;
                in >> bits;
                const u32 mask = (1u << bits) - 1u;
                u32 c = 0;
                while (c < p3::Fp<F>::P && !p3::transcript_is_witness<H>(st, c, mask)) c++;
                if (c == p3::Fp<F>::P) { ok = false; return; }
                const u32 w = p3::to_monty<F>(c);
                u32 s;
                p3::transcript_observe<H, F, true>(st, &w, 1);
                p3::transcript_sample<H, F>(st, &s, 1, true, mask);
                if (s != 0) { ok = false; return; }
                printf("%u\n", w);
            } else {
                ok = false;
            }
        });
        if (!ok) return 2;
        fflush(stdout);
    }
    return 0;
}
