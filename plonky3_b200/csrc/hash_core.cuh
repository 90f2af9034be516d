// The hash primitives of the hot path as device functions: Poseidon2 over the 31-bit Montgomery fields (width 16 / 24),
// Keccak-f[1600] and the SHA-256 compression, and the byte transcript over Keccak-256 or SHA-256.  Kept apart from the kernels
// (hash.cu, challenger.cu) so that the same source can also be compiled as plain C++ and executed on the host against the CPU
// oracle (tests/cpp/hash_core_host.cpp, keccak256_host.cpp, sha256_host.cpp, transcript_host.cpp): g++ ignores the CUDA
// attributes, and the intrinsics used here get host bodies there.
#pragma once
#include "field.cuh"
#include "poseidon2_consts.h"

namespace p3 {

// =================================================================================================
// Poseidon2
// =================================================================================================
// Montgomery product left in (0, 2p): hi(ab) - hi(t p) + p is one IADD3, no conditional correction.  Safe as ONE factor of
// a following product (2p * p < p * 2^32), which then returns to the canonical range.
template <int F> __device__ __forceinline__ u32 mont_mul_lazy(u32 a, u32 b) { return mont_redc_lazy<F>((u64)a * b) + Fp<F>::P; }

template <int F> __device__ __forceinline__ u32 sbox(u32 x) {
    if (Fp<F>::SBOX_D == 3) return mont_mul<F>(mont_mul_lazy<F>(x, x), x);          // x^3: the square stays lazy
    const u32 x2 = mont_mul<F>(x, x);                                                // x^7 = x^4 * x^3, x^3 lazy
    const u32 x3 = mont_mul_lazy<F>(x2, x);
    const u32 x4 = mont_mul<F>(x2, x2);
    return mont_mul<F>(x4, x3);
}

// poseidon2/src/external.rs:60-74: circ(2,3,1,1)
template <int F> __device__ __forceinline__ void mat4(u32 &x0, u32 &x1, u32 &x2, u32 &x3) {
    const u32 t01 = fp_add<F>(x0, x1), t23 = fp_add<F>(x2, x3);
    const u32 t0123 = fp_add<F>(t01, t23);
    const u32 t01123 = fp_add<F>(t0123, x1), t01233 = fp_add<F>(t0123, x3);
    const u32 n3 = fp_add<F>(t01233, fp_double<F>(x0));
    const u32 n1 = fp_add<F>(t01123, fp_double<F>(x2));
    const u32 n0 = fp_add<F>(t01123, t01);
    const u32 n2 = fp_add<F>(t01233, t23);
    x0 = n0; x1 = n1; x2 = n2; x3 = n3;
}
// poseidon2/src/external.rs:113-159
template <int F, int W> __device__ __forceinline__ void mds_light(u32 (&s)[W]) {
#pragma unroll
    for (int i = 0; i < W; i += 4) mat4<F>(s[i], s[i + 1], s[i + 2], s[i + 3]);
    u32 sums[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        sums[k] = s[k];
#pragma unroll
        for (int j = 4; j < W; j += 4) sums[k] = fp_add<F>(sums[k], s[j + k]);
    }
#pragma unroll
    for (int i = 0; i < W; i++) s[i] = fp_add<F>(s[i], sums[i & 3]);
}

// Internal diagonal V (1 + Diag(V) is the internal matrix): koala-bear/src/poseidon2.rs:407-461,
// baby-bear/src/poseidon2.rs:394-450.  Encoded as (mul, shift): V_i = mul * 2^shift, shift <= 0.
struct DiagEntry { int mul, shift; };
template <int F, int W> struct Diag;
template <> struct Diag<BABY_BEAR, 16> { static __host__ __device__ constexpr DiagEntry at(int i) {
    constexpr DiagEntry d[16] = {{-2,0},{1,0},{2,0},{1,-1},{3,0},{4,0},{-1,-1},{-3,0},{-4,0},{1,-8},{1,-2},{1,-3},{1,-27},{-1,-8},{-1,-4},{-1,-27}};
    return d[i]; } };
template <> struct Diag<BABY_BEAR, 24> { static __host__ __device__ constexpr DiagEntry at(int i) {
    constexpr DiagEntry d[24] = {{-2,0},{1,0},{2,0},{1,-1},{3,0},{4,0},{-1,-1},{-3,0},{-4,0},{1,-8},{1,-2},{1,-3},{1,-4},{1,-7},{1,-9},{1,-27},{-1,-8},{-1,-2},{-1,-3},{-1,-4},{-1,-5},{-1,-6},{-1,-7},{-1,-27}};
    return d[i]; } };
template <> struct Diag<KOALA_BEAR, 16> { static __host__ __device__ constexpr DiagEntry at(int i) {
    constexpr DiagEntry d[16] = {{-2,0},{1,0},{2,0},{1,-1},{3,0},{4,0},{-1,-1},{-3,0},{-4,0},{1,-8},{1,-3},{1,-24},{-1,-8},{-1,-3},{-1,-4},{-1,-24}};
    return d[i]; } };
template <> struct Diag<KOALA_BEAR, 24> { static __host__ __device__ constexpr DiagEntry at(int i) {
    constexpr DiagEntry d[24] = {{-2,0},{1,0},{2,0},{1,-1},{3,0},{4,0},{-1,-1},{-3,0},{-4,0},{1,-8},{1,-2},{1,-3},{1,-4},{1,-5},{1,-6},{1,-24},{-1,-8},{-1,-3},{-1,-4},{-1,-5},{-1,-6},{-1,-7},{-1,-9},{-1,-24}};
    return d[i]; } };

// x * 2^-k (monty-31 div_2exp_u64).  Both primes are p = 2^31 - 2^L + 1 (L = 24 KoalaBear, 27 BabyBear), so p = 1 mod 2^k for
// k <= L and the exact quotient is (x + m*p) >> k with m = (-x) mod 2^k:
//     x / 2^k = ceil(x / 2^k) + m * (2^(31-k) - 2^(L-k))            (result < p for x < p)
// = 2 logic/shift ops + 1 add + 1 IMAD, no IMAD.HI (a Montgomery reduction of x << (32-k) costs IMAD + IMAD.HI + 4 ALU ops).
// It is representation-independent: dividing the Montgomery form by 2^k divides the value by 2^k.
template <int F, int K> __device__ __forceinline__ u32 div_2exp(u32 x) {
    constexpr int L = (F == KOALA_BEAR) ? 24 : 27;
    static_assert(K >= 1 && K <= L, "shift exceeds the 2-adic part of p - 1");
    constexpr u32 mask = (1u << K) - 1u;
    constexpr u32 C = (1u << (31 - K)) - (1u << (L - K));
    const u32 m = (0u - x) & mask;
    const u32 c = (x + mask) >> K;
    return c + m * C;
}
template <int F, int W, int I> __device__ __forceinline__ u32 diag_mul_add(u32 x, u32 sum) {
    constexpr DiagEntry d = Diag<F, W>::at(I);
    constexpr int am = d.mul < 0 ? -d.mul : d.mul;
    u32 v;
    if constexpr (d.shift == 0) {
        v = x;
        if (am == 2) v = fp_double<F>(x);
        if (am == 3) v = fp_add<F>(fp_double<F>(x), x);
        if (am == 4) v = fp_double<F>(fp_double<F>(x));
    } else {
        v = div_2exp<F, -d.shift>(x);   // also covers the halves (k = 1)
    }
    return d.mul < 0 ? fp_sub<F>(sum, v) : fp_add<F>(sum, v);
}
template <int F, int W, int I> struct DiagLoop {
    static __device__ __forceinline__ void run(u32 (&s)[W], u32 sum) {
        s[I] = diag_mul_add<F, W, I>(s[I], sum);
        DiagLoop<F, W, I + 1>::run(s, sum);
    }
};
template <int F, int W> struct DiagLoop<F, W, W> { static __device__ __forceinline__ void run(u32 (&)[W], u32) {} };

// One copy of the external-round body and one of the internal-round body (rounds are loops, not unrolled): the fully
// unrolled permutation is 50-300 KB of SASS and the leaf kernels then stall on instruction fetch (ncu: stall_no_instruction
// was the top reason); looped, a whole sponge kernel is 10-20 KB and stays resident in the instruction cache.
template <int F, int W>
__device__ __forceinline__ void poseidon2_permute(u32 (&s)[W], const Poseidon2Consts &k) {
    mds_light<F, W>(s);
#pragma unroll 1
    for (int r = 0; r < 8; r++) {
        if (r == 4) {
            // monty-31/src/poseidon2.rs:76-85
#pragma unroll 1
            for (int q = 0; q < k.rounds_p; q++) {
                s[0] = sbox<F>(fp_add<F>(s[0], k.rc_int[q]));
                u32 part = s[1];
#pragma unroll
                for (int i = 2; i < W; i++) part = fp_add<F>(part, s[i]);
                const u32 sum = fp_add<F>(part, s[0]);
                s[0] = fp_sub<F>(part, s[0]);
                DiagLoop<F, W, 1>::run(s, sum);
            }
        }
        // external round r (0-3 initial, 4-7 terminal): poseidon2/src/external.rs:288-336
#pragma unroll
        for (int i = 0; i < W; i++) s[i] = sbox<F>(fp_add<F>(s[i], k.rc_ext[r * W + i]));
        mds_light<F, W>(s);
    }
}

// =================================================================================================
// Keccak-f[1600]
// =================================================================================================
// The state is kept as 25 (lo, hi) pairs of 32-bit registers: every 64-bit rotation is two funnel shifts (SHF), theta's
// column parity + application and chi are single 3-input LOP3s, so a round is exactly 122 LOP3 + 58 SHF and no register
// moves (the compiler's 64-bit version needed 162 LOP3 + 52 SHF + 46 moves).  All of it runs on the ALU pipe: the kernel is
// bound by that pipe (ncu: 98 % busy).  The (lo, hi) split also matches the leaf packing, which pairs consecutive u32
// field elements into one u64 word (field/src/integers.rs:494-509): lo = first element, hi = second.
static __constant__ u32 KECCAK_RC_LO[24] = {0x00000001u, 0x00008082u, 0x0000808au, 0x80008000u, 0x0000808bu, 0x80000001u, 0x80008081u, 0x00008009u,
                                      0x0000008au, 0x00000088u, 0x80008009u, 0x8000000au, 0x8000808bu, 0x0000008bu, 0x00008089u, 0x00008003u,
                                      0x00008002u, 0x00000080u, 0x0000800au, 0x8000000au, 0x80008081u, 0x00008080u, 0x80000001u, 0x80008008u};
static __constant__ u32 KECCAK_RC_HI[24] = {0x00000000u, 0x00000000u, 0x80000000u, 0x80000000u, 0x00000000u, 0x00000000u, 0x80000000u, 0x80000000u,
                                      0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x80000000u, 0x80000000u, 0x80000000u,
                                      0x80000000u, 0x80000000u, 0x00000000u, 0x80000000u, 0x80000000u, 0x80000000u, 0x00000000u, 0x80000000u};

// 64-bit rotate-left of (lo, hi) by the compile-time constant R
template <int R> __device__ __forceinline__ void rot64(u32 lo, u32 hi, u32 &olo, u32 &ohi) {
    if constexpr (R == 0) { olo = lo; ohi = hi; }
    else if constexpr (R == 32) { olo = hi; ohi = lo; }
    else if constexpr (R < 32) { olo = __funnelshift_l(hi, lo, R); ohi = __funnelshift_l(lo, hi, R); }
    else { olo = __funnelshift_l(lo, hi, R - 32); ohi = __funnelshift_l(hi, lo, R - 32); }
}

struct KState { u32 lo[25], hi[25]; };

__device__ __forceinline__ void keccak_f(KState &s) {
    u32 (&al)[25] = s.lo;
    u32 (&ah)[25] = s.hi;
#pragma unroll 1
    for (int round = 0; round < 24; round++) {
        u32 cl[5], ch[5], rl[5], rh[5];
#pragma unroll
        for (int x = 0; x < 5; x++) {
            cl[x] = al[x] ^ al[x + 5] ^ al[x + 10] ^ al[x + 15] ^ al[x + 20];
            ch[x] = ah[x] ^ ah[x + 5] ^ ah[x + 10] ^ ah[x + 15] ^ ah[x + 20];
        }
#pragma unroll
        for (int x = 0; x < 5; x++) rot64<1>(cl[x], ch[x], rl[x], rh[x]);
        u32 bl[25], bh[25];
        // theta + rho + pi: b[pi(i)] = rotl(a[i] ^ C[x-1] ^ rotl(C[x+1], 1), rho(i))
#define P3_TH(i, R, dst)                                                                             \
    rot64<R>(al[i] ^ cl[((i) % 5 + 4) % 5] ^ rl[((i) % 5 + 1) % 5], ah[i] ^ ch[((i) % 5 + 4) % 5] ^ rh[((i) % 5 + 1) % 5], \
             bl[dst], bh[dst])
        P3_TH(0, 0, 0);
        P3_TH(1, 1, 10);   P3_TH(2, 62, 20);  P3_TH(3, 28, 5);   P3_TH(4, 27, 15);
        P3_TH(5, 36, 16);  P3_TH(6, 44, 1);   P3_TH(7, 6, 11);   P3_TH(8, 55, 21);
        P3_TH(9, 20, 6);   P3_TH(10, 3, 7);   P3_TH(11, 10, 17); P3_TH(12, 43, 2);
        P3_TH(13, 25, 12); P3_TH(14, 39, 22); P3_TH(15, 41, 23); P3_TH(16, 45, 8);
        P3_TH(17, 15, 18); P3_TH(18, 21, 3);  P3_TH(19, 8, 13);  P3_TH(20, 18, 14);
        P3_TH(21, 2, 24);  P3_TH(22, 61, 9);  P3_TH(23, 56, 19); P3_TH(24, 14, 4);
#undef P3_TH
#pragma unroll
        for (int y = 0; y < 5; y++)
#pragma unroll
            for (int x = 0; x < 5; x++) {
                al[x + 5 * y] = bl[x + 5 * y] ^ (~bl[(x + 1) % 5 + 5 * y] & bl[(x + 2) % 5 + 5 * y]);
                ah[x + 5 * y] = bh[x + 5 * y] ^ (~bh[(x + 1) % 5 + 5 * y] & bh[(x + 2) % 5 + 5 * y]);
            }
        al[0] ^= KECCAK_RC_LO[round];
        ah[0] ^= KECCAK_RC_HI[round];
    }
}

// =================================================================================================
// Keccak-256 (keccak/src/lib.rs Keccak256Hash = tiny-keccak Keccak::v256)
// =================================================================================================
// Rate 136 bytes, Keccak's original padding: 0x01 after the message and 0x80 OR'd into the last byte of the block (not SHA3's
// 0x06).  Blocks are handled as 34 little-endian 32-bit words, word 2i / 2i + 1 being lane i's lo / hi half.  Every transcript
// input is a whole number of words (4-byte field elements, 32-byte digests), so the transcript (challenger.cu) uses the word
// functions; `keccak256` hashes any byte string and is the host tests' entry point.
constexpr int KECCAK256_RATE_WORDS = 34;

__device__ __forceinline__ void keccak256_absorb_block(KState &s, const u32 (&w)[KECCAK256_RATE_WORDS]) {
#pragma unroll
    for (int i = 0; i < KECCAK256_RATE_WORDS / 2; i++) { s.lo[i] ^= w[2 * i]; s.hi[i] ^= w[2 * i + 1]; }
    keccak_f(s);
}

// The last block: the first n < 34 words of `w` hold the message tail (the rest is ignored); padding is added and the block
// absorbed.  The digest is then words 0..7 = lo[0], hi[0], ..., lo[3], hi[3].  Static indices only, so the block stays in
// registers.
__device__ __forceinline__ void keccak256_final_block(KState &s, const u32 (&w)[KECCAK256_RATE_WORDS], u32 n) {
    u32 b[KECCAK256_RATE_WORDS];
#pragma unroll
    for (int i = 0; i < KECCAK256_RATE_WORDS; i++) b[i] = ((u32)i < n ? w[i] : 0u) ^ ((u32)i == n ? 0x01u : 0u);
    b[KECCAK256_RATE_WORDS - 1] ^= 0x80000000u;
    keccak256_absorb_block(s, b);
}

__device__ __forceinline__ u32 keccak256_digest_word(const KState &s, int k) { return (k & 1) ? s.hi[k >> 1] : s.lo[k >> 1]; }

__device__ inline void keccak256(const unsigned char *msg, size_t len, unsigned char out[32]) {
    KState s;
#pragma unroll
    for (int i = 0; i < 25; i++) { s.lo[i] = 0; s.hi[i] = 0; }
    u32 w[KECCAK256_RATE_WORDS];
    size_t off = 0;
    for (;;) {
        const size_t n = len - off < 136 ? len - off : 136;
        for (int i = 0; i < KECCAK256_RATE_WORDS; i++) w[i] = 0;
        for (size_t j = 0; j < n; j++) w[j >> 2] |= (u32)msg[off + j] << (8 * (j & 3));
        off += n;
        if (n == 136) { keccak256_absorb_block(s, w); continue; }
        w[n >> 2] ^= 0x01u << (8 * (n & 3));                  // padding inside a partly filled word
        w[KECCAK256_RATE_WORDS - 1] ^= 0x80000000u;
        keccak256_absorb_block(s, w);
        break;
    }
    for (int k = 0; k < 8; k++) {
        const u32 v = keccak256_digest_word(s, k);
        for (int j = 0; j < 4; j++) out[4 * k + j] = (unsigned char)(v >> (8 * j));
    }
}

// =================================================================================================
// SHA-256 (FIPS 180-4; sha256/src/lib.rs Sha256 = sha2::Sha256, Sha256Compress = one compress256 from H256_256)
// =================================================================================================
// The 64 rounds and the 48 schedule words are fully unrolled: the round constants become constant-bank operands and the 16-word
// schedule window stays in registers under static indices.  A round is 3 funnel-shift rotations + 1 LOP3 for each of Sigma0 and
// Sigma1, one LOP3 each for Ch and Maj and three IADD3s; a schedule word 2 rotations + 1 shift + 1 LOP3 for each of sigma0 and
// sigma1 and two IADD3s.  All of it is integer-ALU work.  Message words are big-endian: a 32-bit word holding 4 stream bytes in
// little-endian order (a field element's bytes, a digest word) enters the block byte-swapped.
static __constant__ u32 SHA256_K[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, 0xd807aa98u, 0x12835b01u,
    0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, 0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu,
    0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, 0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u,
    0x06ca6351u, 0x14292967u, 0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u, 0x19a4c116u, 0x1e376c08u,
    0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u,
    0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
// The initial hash value; a function so that host code (the transcript's initial state) reads the same constants
__host__ __device__ constexpr u32 sha256_iv_word(int i) {
    constexpr u32 iv[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    return iv[i];
}
// the copy the hash kernels read, as constant-bank operands
static __constant__ u32 SHA256_IV[8] = {sha256_iv_word(0), sha256_iv_word(1), sha256_iv_word(2), sha256_iv_word(3),
                                        sha256_iv_word(4), sha256_iv_word(5), sha256_iv_word(6), sha256_iv_word(7)};

__device__ __forceinline__ u32 rotr32(u32 x, int r) { return __funnelshift_l(x, x, 32 - r); }
__device__ __forceinline__ u32 bswap32(u32 x) {
#ifdef __CUDA_ARCH__
    return __byte_perm(x, 0, 0x0123);
#else
    return __builtin_bswap32(x);
#endif
}
__device__ __forceinline__ void sha256_iv(u32 (&st)[8]) {
#pragma unroll
    for (int i = 0; i < 8; i++) st[i] = SHA256_IV[i];
}

// compress256: st = st + rounds(st, block w) for one 16-word big-endian block
__device__ __forceinline__ void sha256_compress(u32 (&st)[8], const u32 (&win)[16]) {
    u32 w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = win[i];
    u32 a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int r = 0; r < 64; r++) {
        const int i = r & 15;
        if (r >= 16) {
            const u32 w15 = w[(i + 1) & 15], w2 = w[(i + 14) & 15];
            const u32 s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
            const u32 s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
            w[i] = w[i] + s0 + w[(i + 9) & 15] + s1;
        }
        const u32 S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
        const u32 ch = (e & f) ^ (~e & g);
        const u32 t1 = h + S1 + ch + SHA256_K[r] + w[i];
        const u32 S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
        const u32 maj = (a & b) ^ (a & c) ^ (b & c);
        h = g; g = f; f = e; e = d + t1;
        d = c; c = b; b = a; a = t1 + S0 + maj;
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// Word j (j >= n) of the padding after the last n message words, which fill nb blocks with it: 0x80 right after the message (a whole
// word: every input is a whole number of words), zeros, then the whole message's bit length `bits` as a big-endian u64 in the last
// two words of block nb - 1.
__device__ __forceinline__ u32 sha256_pad_word(u64 j, u64 n, u64 nb, u64 bits) {
    if (j == n) return 0x80000000u;
    if (j == 16 * nb - 2) return (u32)(bits >> 32);
    if (j == 16 * nb - 1) return (u32)bits;
    return 0u;
}
// blocks of a padded message of n words: room for the 0x80 word and the two length words
__device__ __forceinline__ u64 sha256_blocks(u64 n) { return (n + 2) / 16 + 1; }

// SHA-256 of any byte string (the host tests' entry point)
__device__ inline void sha256(const unsigned char *msg, size_t len, unsigned char out[32]) {
    u32 st[8];
    sha256_iv(st);
    const size_t nb = (len + 9 + 63) / 64;
    for (size_t blk = 0; blk < nb; blk++) {
        unsigned char b[64];
        for (int i = 0; i < 64; i++) {
            const size_t j = blk * 64 + i;
            b[i] = j < len ? msg[j] : (j == len ? 0x80 : 0);
        }
        if (blk == nb - 1) for (int i = 0; i < 8; i++) b[56 + i] = (unsigned char)(((u64)len * 8) >> (56 - 8 * i));
        u32 w[16];
        for (int i = 0; i < 16; i++) w[i] = (u32)b[4 * i] << 24 | (u32)b[4 * i + 1] << 16 | (u32)b[4 * i + 2] << 8 | b[4 * i + 3];
        sha256_compress(st, w);
    }
    for (int k = 0; k < 8; k++)
        for (int j = 0; j < 4; j++) out[4 * k + j] = (unsigned char)(st[k] >> (24 - 8 * j));
}

// =================================================================================================
// SerializingChallenger32<F, HashChallenger<u8, H, 32>> (challenger/src/serializing_challenger.rs, hash_challenger.rs)
// =================================================================================================
// The transcript of the Keccak and SHA-256 configurations.  The reference keeps every observed byte in an input buffer and hashes
// all of it when a sample finds the output buffer empty; the digest then becomes both the new input buffer and the output buffer,
// whose bytes are popped from the end.  Absorbing the input block by block as it fills gives the same digest, so the state is the
// hash's running state over the full blocks plus the pending words of the partial block; every input is a whole number of 32-bit
// words (4-byte field elements, 32-byte digests).  The state is an array of TR_WORDS words (device memory in challenger.cu, a host
// array in tests/cpp/transcript_host.cpp):
//     [0, 64)              the hash's running state, laid out by the policy
//     [TR_PEND, +BLOCK)    the pending words, in the hash's block representation; [TR_NPEND] their number
//     [TR_OUT, +8)         the output buffer: the digest as 8 big-endian words, so that the u32 of the 4 bytes popped off its end
//                          (u32::from_le_bytes of bytes 4m+3, 4m+2, 4m+1, 4m) is word m itself; [TR_NOUT] how many words are left
// A policy gives the block size in words, the running State (held in registers) with init / load / store over the state words,
// absorb (one full block), finish (the pending words, an optional extra word and the padding: the digest as big-endian words) and
// block_word (a word of 4 stream bytes in little-endian order, as it enters a block).  absorb and finish also see the state words,
// for what a policy keeps there rather than in registers.
constexpr int TR_PEND = 64, TR_NPEND = 98, TR_OUT = 100, TR_NOUT = 108, TR_WORDS = 128;

// Keccak256Hash: the Keccak state as (lo[25], hi[25]) at [0, 50), zero initially; 34-word blocks of little-endian words
struct Keccak256Policy {
    static constexpr int BLOCK = KECCAK256_RATE_WORDS;
    typedef KState State;
    static __host__ __device__ void init(u32 *st) {
        for (int i = 0; i < 50; i++) st[i] = 0;
    }
    static __device__ __forceinline__ void load(const u32 *st, State &s) {
#pragma unroll
        for (int i = 0; i < 25; i++) { s.lo[i] = st[i]; s.hi[i] = st[25 + i]; }
    }
    static __device__ __forceinline__ void store(u32 *st, const State &s) {
#pragma unroll
        for (int i = 0; i < 25; i++) { st[i] = s.lo[i]; st[25 + i] = s.hi[i]; }
    }
    static __device__ __forceinline__ u32 block_word(u32 x) { return x; }
    static __device__ __forceinline__ void absorb(u32 *, State &s, const u32 (&w)[BLOCK]) { keccak256_absorb_block(s, w); }
    // the n < BLOCK pending words, then `extra` if has_extra: one Keccak-f, or two when the extra word completes the block
    static __device__ __forceinline__ void finish(State &s, const u32 *st, bool has_extra, u32 extra, u32 (&d)[8]) {
        const u32 n = st[TR_NPEND], *pend = st + TR_PEND;
        u32 w[BLOCK];
#pragma unroll
        for (int i = 0; i < BLOCK; i++) w[i] = (u32)i < n ? pend[i] : (has_extra && (u32)i == n ? extra : 0u);
        u32 tail = n + (has_extra ? 1u : 0u);
        if (tail == (u32)BLOCK) { keccak256_absorb_block(s, w); tail = 0; }
        keccak256_final_block(s, w, tail);
#pragma unroll
        for (int k = 0; k < 8; k++) d[k] = bswap32(keccak256_digest_word(s, k));
    }
};

// Sha256: the midstate at [0, 8) (the IV initially) and the number of full blocks at [8] (for the length in the padding);
// 16-word blocks of big-endian words.  The block count stays in the state words, not in State: held in a register it made ptxas
// schedule the single-thread observe kernel's compression 7 % slower (H100 80GB HBM3, 700 W); in memory the kernel is unchanged.
struct Sha256Policy {
    static constexpr int BLOCK = 16;
    struct State { u32 h[8]; };
    static __host__ __device__ void init(u32 *st) {
        for (int i = 0; i < 8; i++) st[i] = sha256_iv_word(i);
        st[8] = 0;
    }
    static __device__ __forceinline__ void load(const u32 *st, State &s) {
#pragma unroll
        for (int i = 0; i < 8; i++) s.h[i] = st[i];
    }
    static __device__ __forceinline__ void store(u32 *st, const State &s) {
#pragma unroll
        for (int i = 0; i < 8; i++) st[i] = s.h[i];
    }
    static __device__ __forceinline__ u32 block_word(u32 x) { return bswap32(x); }
    static __device__ __forceinline__ void absorb(u32 *st, State &s, const u32 (&w)[BLOCK]) { sha256_compress(s.h, w); st[8]++; }
    // the n < BLOCK pending words, then `extra` if has_extra, then the padding: one or two compressions through one inlined copy of
    // the compression
    static __device__ __forceinline__ void finish(State &s, const u32 *st, bool has_extra, u32 extra, u32 (&d)[8]) {
        const u32 n = st[TR_NPEND], *pend = st + TR_PEND;
        const u32 tail = n + (has_extra ? 1u : 0u);
        const u64 nb = sha256_blocks(tail), bits = ((u64)st[8] * 16 + tail) * 32;
#pragma unroll 1
        for (u64 b = 0; b < nb; b++) {
            u32 w[16];
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const u64 j = 16 * b + i;
                w[i] = j < n ? pend[i] : (j < tail ? extra : sha256_pad_word(j, tail, nb, bits));
            }
            sha256_compress(s.h, w);
        }
#pragma unroll
        for (int k = 0; k < 8; k++) d[k] = s.h[k];
    }
};

// CanObserve.  MONTY: Montgomery words, observed as the 4 little-endian bytes of their canonical values (CanObserve<F>); otherwise
// words observed as their own bytes (a digest held as 8 words).  Any buffered output is invalidated.
template <class H, int F, bool MONTY>
__device__ void transcript_observe(u32 *st, const u32 *vals, size_t n) {
    if (n == 0) return;
    typename H::State s;
    H::load(st, s);
    st[TR_NOUT] = 0;
    u32 m = st[TR_NPEND];
    for (size_t j = 0; j < n; j++) {
        st[TR_PEND + m] = H::block_word(MONTY ? from_monty<F>(vals[j]) : vals[j]);
        if (++m == (u32)H::BLOCK) {
            u32 w[H::BLOCK];
#pragma unroll
            for (int i = 0; i < H::BLOCK; i++) w[i] = st[TR_PEND + i];
            H::absorb(st, s, w);
            m = 0;
        }
    }
    st[TR_NPEND] = m;
    H::store(st, s);
}

// HashChallenger::flush: the digest of everything observed is the new input buffer (the running state back at its start) and the
// output buffer
template <class H>
__device__ void transcript_flush(u32 *st) {
    typename H::State s;
    H::load(st, s);
    u32 d[8];
    H::finish(s, st, false, 0u, d);
    H::init(st);
#pragma unroll
    for (int k = 0; k < 8; k++) { st[TR_PEND + k] = H::block_word(bswap32(d[k])); st[TR_OUT + k] = d[k]; }
    st[TR_NPEND] = 8;
    st[TR_NOUT] = 8;
}

// Four bytes popped from the END of the output buffer, as u32::from_le_bytes of the popped order: the last big-endian word left
template <class H>
__device__ __forceinline__ u32 transcript_pop_u32(u32 *st) {
    if (st[TR_NOUT] == 0) transcript_flush<H>(st);
    const u32 m = st[TR_NOUT] - 1;
    st[TR_NOUT] = m;
    return st[TR_OUT + m];
}

// raw = false: n field elements by rejection sampling of 31-bit values (CanSample<F>), as Montgomery words; raw = true: n u32s of
// 4 popped bytes AND `mask` (CanSampleBits)
template <class H, int F>
__device__ void transcript_sample(u32 *st, u32 *out, size_t n, bool raw, u32 mask) {
    for (size_t j = 0; j < n; j++) {
        if (raw) { out[j] = transcript_pop_u32<H>(st) & mask; continue; }
        u32 v;
        do { v = transcript_pop_u32<H>(st) & 0x7fffffffu; } while (v >= Fp<F>::P);
        out[j] = to_monty<F>(v);
    }
}

// Whether the canonical value c is a proof-of-work witness: observe(c); sample_bits(bits) == 0 (mask = 2^bits - 1), read off
// without changing the state.  The hash is finished from the running state with the pending words and c; the first sampled u32
// is the last big-endian digest word.
template <class H>
__device__ __forceinline__ bool transcript_is_witness(const u32 *st, u32 c, u32 mask) {
    typename H::State s;
    H::load(st, s);
    u32 d[8];
    H::finish(s, st, true, H::block_word(c), d);
    return (d[7] & mask) == 0;
}

}  // namespace p3
