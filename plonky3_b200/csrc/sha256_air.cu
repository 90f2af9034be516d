// SHA-256 AIR on the device: trace generation and quotient evaluation for the reference's Sha256Air (sha256-air/src), one SHA-256
// compression per row, over BabyBear and KoalaBear.
//
//   trace generation   sha256-air/src/generation.rs: row i compresses its 24 input words (the 16-word block, then the 8-word
//                      chaining state); 7728 columns
//   constraints        sha256-air/src/air.rs + air/src/utils.rs (add2, add3, pack_bits_le): 8096 constraints of degree <= 3 on the
//                      local row only, folded with alpha^(8095 - k) in eval order
//   quotient           uni-stark/src/prover.rs:462-827 over GENERATOR * K, |K| = 2 N (two quotient chunks), times 1 / Z_H
//
// Column layout (columns.rs Sha256Cols, repr(C)); bits least significant first, limbs [lo, hi]:
//   h_in [8][2] [0,16) | a_chain [68][32] [16,2192) | e_chain [68][32] [2192,4368) | w [64][32] [4368,6416) |
//   sched_sigma0, sched_sigma1, sched_tmp [48][2] each [6416,6704) | rounds [64] x (sigma1_e, ch, tmp1, t1, sigma0_a, maj) [2] each
//   [6704,7472) | h_out [8][32] [7472,7728)
// a_chain[0..4] = H3, H2, H1, H0 and a_chain[t + 4] = new_a of round t (e_chain likewise with H7..H4, new_e), so round t reads
// a, b, c, d = a_chain[t + 3], [t + 2], [t + 1], [t].
#include "common.h"
#include "air_program.cuh"

namespace p3 {

constexpr int SH_COLS = 7728, SH_CONSTRAINTS = 8096;
constexpr int SH_H_IN = 0, SH_A = 16, SH_E = 2192, SH_W = 4368, SH_SIG0 = 6416, SH_SIG1 = 6512, SH_TMP = 6608, SH_ROUNDS = 6704, SH_H_OUT = 7472;
// constraint indices: booleans of w, a_chain, e_chain, h_out (in that order, not column order), the h_in bridges, 48 schedule
// steps of 8, 64 rounds of 16, the finalization
constexpr int SH_K_BOOL_A = 2048, SH_K_BOOL_E = 4224, SH_K_BOOL_OUT = 6400, SH_K_HIN = 6656, SH_K_SCHED = 6672, SH_K_ROUND = 7056,
              SH_K_FINAL = 8080;

__constant__ u32 SH_K[64] = {
    0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, 0xd807aa98u, 0x12835b01u,
    0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, 0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu,
    0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau, 0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u,
    0x06ca6351u, 0x14292967u, 0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
    0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u, 0x19a4c116u, 0x1e376c08u,
    0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u,
    0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};

__device__ __forceinline__ u32 sh_rotr(u32 v, int r) { return __funnelshift_r(v, v, r); }

// ---- trace generation -----------------------------------------------------------------------------------------------------
// One warp per row.  Every lane runs the compression in registers: the working variables are warp-uniform, and the message
// schedule is lane-distributed (lane l holds W[l] and W[32 + l]; W[j] is one shuffle away).  Lane l owns bit l of every word, so
// a bit array is one 128-byte store per warp instruction; the packed limbs of a schedule step (6) or a round (12) are one store by
// the low lanes.  Nothing is read but the row's 96-byte input.
// WINDOW: only columns [win.col0, win.col1) are stored, as a dense n x (col1 - col0) matrix: the column block one rank of the sharded
// prover commits.  The whole compression still runs; only the stores are filtered.
constexpr int SG_WARPS = 8;

template <int F, bool WINDOW>
__global__ void __launch_bounds__(32 * SG_WARPS) sha256_air_generate_kernel(const u32 *inputs, size_t n, u32 *trace, const GenWindow win) {
    const unsigned lane = threadIdx.x & 31u;
    const size_t row = (size_t)blockIdx.x * SG_WARPS + (threadIdx.x >> 5);
    if (row >= n) return;
    const u32 ONE = Fp<F>::ONE;
    const u32 word = lane < 24 ? __ldg(inputs + row * 24 + lane) : 0u;
    u32 *out = WINDOW ? trace + row * (win.col1 - win.col0) : trace + row * SH_COLS;
    auto put = [&](int c, u32 v) {
        if constexpr (WINDOW) {
            if ((size_t)c >= win.col0 && (size_t)c < win.col1) out[c - win.col0] = v;
        } else {
            out[c] = v;
        }
    };
    auto bits = [&](int col, u32 w) { put(col + lane, (w >> lane) & 1u ? ONE : 0u); };
    auto limb = [](u32 w, unsigned hi) { return to_monty<F>(hi ? w >> 16 : w & 0xffffu); };
    u32 h[8];
#pragma unroll
    for (int j = 0; j < 8; j++) h[j] = __shfl_sync(0xffffffffu, word, 16 + j);
    {
        const u32 hw = __shfl_sync(0xffffffffu, word, 16 + ((lane >> 1) & 7u));   // lane l < 16: limb l & 1 of H[l >> 1]
        if (lane < 16) put(SH_H_IN + lane, limb(hw, lane & 1u));
    }
    // message schedule (generation.rs step 2)
    u32 w0 = lane < 16 ? word : 0u, w1 = 0u;
    auto wget = [&](int j) { return __shfl_sync(0xffffffffu, j < 32 ? w0 : w1, j & 31); };
#pragma unroll
    for (int j = 0; j < 16; j++) bits(SH_W + 32 * j, __shfl_sync(0xffffffffu, word, j));
#pragma unroll 1
    for (int t = 16; t < 64; t++) {
        const u32 x15 = wget(t - 15), x2 = wget(t - 2);
        const u32 s0 = sh_rotr(x15, 7) ^ sh_rotr(x15, 18) ^ (x15 >> 3);
        const u32 s1 = sh_rotr(x2, 17) ^ sh_rotr(x2, 19) ^ (x2 >> 10);
        const u32 tmp = s1 + wget(t - 7);
        const u32 wt = tmp + s0 + wget(t - 16);
        if (lane == (unsigned)(t & 31)) {
            if (t < 32) w0 = wt; else w1 = wt;
        }
        bits(SH_W + 32 * t, wt);
        if (lane < 6) {                                                 // sched_sigma0[i], sched_sigma1[i], sched_tmp[i], i = t - 16
            const unsigned j = lane >> 1;
            const u32 v = j == 0 ? s0 : j == 1 ? s1 : tmp;
            put((j == 0 ? SH_SIG0 : j == 1 ? SH_SIG1 : SH_TMP) + 2 * (t - 16) + (lane & 1u), limb(v, lane & 1u));
        }
    }
    // compression (generation.rs step 3): the chains' first four slots are (d, c, b, a) = H3..H0 and (h, g, f, e) = H7..H4
#pragma unroll
    for (int j = 0; j < 4; j++) {
        bits(SH_A + 32 * j, h[3 - j]);
        bits(SH_E + 32 * j, h[7 - j]);
    }
    u32 a = h[0], b = h[1], c = h[2], d = h[3], e = h[4], f = h[5], g = h[6], hh = h[7];
#pragma unroll 1
    for (int t = 0; t < 64; t++) {
        const u32 s1e = sh_rotr(e, 6) ^ sh_rotr(e, 11) ^ sh_rotr(e, 25);
        const u32 ch = (e & f) ^ (~e & g);
        const u32 tmp1 = hh + s1e + ch;
        const u32 t1 = tmp1 + SH_K[t] + wget(t);
        const u32 s0a = sh_rotr(a, 2) ^ sh_rotr(a, 13) ^ sh_rotr(a, 22);
        const u32 maj = (a & b) ^ (a & c) ^ (b & c);
        const u32 na = t1 + s0a + maj, ne = d + t1;
        if (lane < 12) {                                                // rounds[t]: sigma1_e, ch, tmp1, t1, sigma0_a, maj
            const unsigned j = lane >> 1;
            const u32 v = j == 0 ? s1e : j == 1 ? ch : j == 2 ? tmp1 : j == 3 ? t1 : j == 4 ? s0a : maj;
            put(SH_ROUNDS + 12 * t + lane, limb(v, lane & 1u));
        }
        bits(SH_A + 32 * (t + 4), na);
        bits(SH_E + 32 * (t + 4), ne);
        hh = g; g = f; f = e; e = ne;
        d = c; c = b; b = a; a = na;
    }
    // finalization (generation.rs step 4)
    const u32 fin[8] = {a, b, c, d, e, f, g, hh};
#pragma unroll
    for (int j = 0; j < 8; j++) bits(SH_H_OUT + 32 * j, h[j] + fin[j]);
}

// ---- quotient -------------------------------------------------------------------------------------------------------------
// One warp per point of the quotient domain, persistent blocks of SQ_WARPS warps, one block per SM (on an H100 at 700 W, 24 warps
// ran the 2^18-row quotient in 50 ms where 16 took 60 ms: more warps hide the shuffle chains' latency).  The block holds the whole
// alpha-power table (alpha^(8095 - k), 129.5 KB) in shared memory, so rows are read from global memory as they are used: a bit array is one
// coalesced 128-byte load (lane l reads bit l), a step's or a round's packed limbs one load by the low lanes, then broadcast.
//   - a boolean check of bit l is lane l's constraint, folded where the word is loaded;
//   - a sigma is three shuffles and two air_bxor per lane; Ch and Maj are lane-local; a 16-bit pack sums the weighted bits over a
//     half warp, and both halves are broadcast;
//   - the limb-level constraints (the packed checks and add2 / add3) are warp-uniform values; lane j keeps the j-th and folds it;
//   - every a / e chain word is loaded and packed once: a 4-deep window of bits and limbs covers its uses as a, b, c and d (e, f,
//     g and h); the 64 schedule words are packed once up front, lane-distributed over four registers.
// Each lane folds its constraints with air_qmac; air_warp_store adds the 32 partial sums and multiplies by 1 / Z_H.
// SHARDED: one rank's chunk-major row block (AirHandQArgs); every column address goes through the unit table behind the alpha
// powers (air_program.cuh AirShardRow), the block's rows are the points, and the quotient lands in the block's slice.
constexpr int SQ_WARPS = 24;
constexpr size_t SQ_SMEM = (size_t)SH_CONSTRAINTS * 16;

template <int F, bool SHARDED> __global__ void __launch_bounds__(32 * SQ_WARPS, 1) sha256_air_quotient_kernel(const AirHandQArgs a) {
    extern __shared__ uint4 sq_sm[];
    const uint4 *ap = sq_sm;
    u64 *units = reinterpret_cast<u64 *>(sq_sm + SH_CONSTRAINTS);
    for (int t = threadIdx.x; t < SH_CONSTRAINTS; t += blockDim.x) sq_sm[t] = __ldg(a.apow + t);
    if constexpr (SHARDED) air_shard_table_load(a, units);
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const u32 n_pts = SHARDED ? a.rows : 1u << a.d.log_q;
    const u32 ONE = Fp<F>::ONE;
    const u32 T16 = to_monty<F>(1u << 16), T17 = fp_double<F>(T16), T32 = mont_mul<F>(T16, T16), T33 = fp_double<F>(T32);
    const u32 wpow = to_monty<F>(1u << (lane & 15u));                  // weight of this lane's bit in its 16-bit limb
    auto add = [](u32 x, u32 y) { return fp_add<F>(x, y); };
    auto sub = [](u32 x, u32 y) { return fp_sub<F>(x, y); };
    auto mul = [](u32 x, u32 y) { return mont_mul<F>(x, y); };
    auto bc = [](u32 v, int src) { return __shfl_sync(0xffffffffu, v, src); };
    // pack_bits_le of the lane-distributed bits v over [0, 16) and [16, 32): (lo, hi), warp-uniform
    auto pack = [&](u32 v, u32 &lo, u32 &hi) {
        u32 s = mul(v, wpow);
#pragma unroll
        for (int o = 8; o; o >>= 1) s = add(s, __shfl_xor_sync(0xffffffffu, s, o));
        lo = bc(s, 0); hi = bc(s, 16);
    };
    // this lane's bit of ROTR_r1(x) ^ ROTR_r2(x) ^ ROTR_r3(x) (SHR_r3(x) if shr): air.rs assert_sigma_matches' xor3
    auto sigma = [&](u32 x, int r1, int r2, int r3, bool shr) {
        const u32 b1 = bc(x, (lane + r1) & 31u), b2 = bc(x, (lane + r2) & 31u), b3 = bc(x, (lane + r3) & 31u);
        return air_bxor<F>(air_bxor<F>(b1, b2), shr && lane + r3 >= 32 ? 0u : b3);
    };
    for (u32 i = blockIdx.x * SQ_WARPS + warp; i < n_pts; i += gridDim.x * SQ_WARPS) {
        const u32 *row = SHARDED ? a.lde : a.lde + (size_t)air_bitrev(i, a.d.log_q) * SH_COLS;
        const AirShardRow sr{a.lde, units, i};
        auto ld = [row, sr](int c) {
            if constexpr (SHARDED) return sr.ld((u32)c);
            else return __ldg(row + c);
        };
        u64 acc[4] = {0, 0, 0, 0};
        auto fold = [&](int k, u32 c) { air_qmac<F>(acc, c, ap[k]); };
        u32 mine = 0;
        // packed == (lo, hi): constraints j, j + 1
        auto eq2 = [&](u32 p0, u32 p1, u32 lo, u32 hi, int j) {
            if (lane == (unsigned)j) mine = sub(p0, lo);
            if (lane == (unsigned)j + 1) mine = sub(p1, hi);
        };
        // add2 / add3 (air/src/utils.rs; the sha256-local _expr_out variants are the same polynomials): x = y + z (+ u) mod 2^32 on
        // [lo, hi] limbs, the 2^32 check at j, the 2^16 check at j + 1
        auto add2 = [&](u32 x0, u32 x1, u32 y0, u32 y1, u32 z0, u32 z1, int j) {
            const u32 acc16 = sub(sub(x0, y0), z0), acc32 = sub(sub(x1, y1), z1);
            const u32 accv = add(acc16, mul(acc32, T16));
            if (lane == (unsigned)j) mine = mul(accv, add(accv, T32));
            if (lane == (unsigned)j + 1) mine = mul(acc16, add(acc16, T16));
        };
        auto add3 = [&](u32 x0, u32 x1, u32 y0, u32 y1, u32 z0, u32 z1, u32 u0, u32 u1, int j) {
            const u32 acc16 = sub(sub(sub(x0, y0), z0), u0), acc32 = sub(sub(sub(x1, y1), z1), u1);
            const u32 accv = add(acc16, mul(acc32, T16));
            if (lane == (unsigned)j) mine = mul(mul(accv, add(accv, T32)), add(accv, T33));
            if (lane == (unsigned)j + 1) mine = mul(mul(acc16, add(acc16, T16)), add(acc16, T17));
        };
        const u32 hin = lane < 16 ? ld(SH_H_IN + lane) : 0u;           // lane l < 16: h_in limb l
        // the schedule words: booleans (k = 32 j + l) and packs; lane l of wp[s] holds limb (l & 1) of w[16 s + (l >> 1)]
        u32 wp[4];
#pragma unroll
        for (int s = 0; s < 4; s++) {
            wp[s] = 0;
#pragma unroll 1
            for (int jj = 0; jj < 16; jj++) {
                const int j = 16 * s + jj;
                const u32 x = ld(SH_W + 32 * j + lane);
                fold(32 * j + lane, air_bool<F>(x));
                u32 lo, hi;
                pack(x, lo, hi);
                if ((lane >> 1) == (unsigned)jj) wp[s] = lane & 1u ? hi : lo;
            }
        }
        auto wpack = [&](int j, u32 &lo, u32 &hi) {
            const int s = j >> 4;
            const u32 src = s == 0 ? wp[0] : s == 1 ? wp[1] : s == 2 ? wp[2] : wp[3];
            lo = bc(src, 2 * (j & 15)); hi = bc(src, 2 * (j & 15) + 1);
        };
        // message schedule, step s (t = s + 16), 8 constraints at SH_K_SCHED + 8 s: small sigma0 (0, 1), small sigma1 (2, 3),
        // add2(tmp, sigma1, pack(w[t - 7])) (4, 5), add3_expr_out(pack(w[t]), tmp, sigma0, pack(w[t - 16])) (6, 7)
#pragma unroll 1
        for (int s = 0; s < 48; s++) {
            const int t = s + 16;
            const unsigned j3 = lane >> 1;
            const u32 lim = lane < 6 ? ld((j3 == 0 ? SH_SIG0 : j3 == 1 ? SH_SIG1 : SH_TMP) + 2 * s + (lane & 1u)) : 0u;
            const u32 s0l = bc(lim, 0), s0h = bc(lim, 1), s1l = bc(lim, 2), s1h = bc(lim, 3), tl = bc(lim, 4), th = bc(lim, 5);
            u32 lo, hi, xl, xh;
            mine = 0;
            pack(sigma(ld(SH_W + 32 * (t - 15) + lane), 7, 18, 3, true), lo, hi);   eq2(s0l, s0h, lo, hi, 0);
            pack(sigma(ld(SH_W + 32 * (t - 2) + lane), 17, 19, 10, true), lo, hi);  eq2(s1l, s1h, lo, hi, 2);
            wpack(t - 7, lo, hi);                                                   add2(tl, th, s1l, s1h, lo, hi, 4);
            wpack(t, xl, xh); wpack(t - 16, lo, hi);                                add3(xl, xh, tl, th, s0l, s0h, lo, hi, 6);
            if (lane < 8) fold(SH_K_SCHED + 8 * s + lane, mine);
        }
        // the chains' first four words: booleans, packs, and h_in[i] = pack(a_chain[3 - i]), h_in[4 + i] = pack(e_chain[3 - i])
        // (k = SH_K_HIN + l for h_in limb l)
        u32 A[4], E[4], al[4], ah[4], el[4], eh[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            A[j] = ld(SH_A + 32 * j + lane); fold(SH_K_BOOL_A + 32 * j + lane, air_bool<F>(A[j])); pack(A[j], al[j], ah[j]);
            E[j] = ld(SH_E + 32 * j + lane); fold(SH_K_BOOL_E + 32 * j + lane, air_bool<F>(E[j])); pack(E[j], el[j], eh[j]);
        }
        mine = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            eq2(hin, hin, al[3 - j], ah[3 - j], 2 * j);
            eq2(hin, hin, el[3 - j], eh[3 - j], 8 + 2 * j);
        }
        if (lane < 16) fold(SH_K_HIN + lane, mine);
        // round t, 16 constraints at SH_K_ROUND + 16 t: sigma1_e (0, 1), ch (2, 3), add3 tmp1 (4, 5), add3 t1 with K[t] (6, 7),
        // sigma0_a (8, 9), maj (10, 11), add3_expr_out new_a (12, 13), add2_expr_out new_e (14, 15)
#pragma unroll 1
        for (int t = 0; t < 64; t++) {
            const u32 lim = lane < 12 ? ld(SH_ROUNDS + 12 * t + lane) : 0u;
            u32 r[12];
#pragma unroll
            for (int j = 0; j < 12; j++) r[j] = bc(lim, j);
            u32 lo, hi;
            mine = 0;
            pack(sigma(E[3], 6, 11, 25, false), lo, hi);                            eq2(r[0], r[1], lo, hi, 0);
            pack(add(mul(E[3], E[2]), mul(sub(ONE, E[3]), E[1])), lo, hi);          eq2(r[2], r[3], lo, hi, 2);
            add3(r[4], r[5], r[0], r[1], r[2], r[3], el[0], eh[0], 4);
            const u32 kt = SH_K[t];
            wpack(t, lo, hi);
            add3(r[6], r[7], r[4], r[5], to_monty<F>(kt & 0xffffu), to_monty<F>(kt >> 16), lo, hi, 6);
            pack(sigma(A[3], 2, 13, 22, false), lo, hi);                            eq2(r[8], r[9], lo, hi, 8);
            pack(add(mul(A[3], A[2]), mul(A[1], air_bxor<F>(A[3], A[2]))), lo, hi); eq2(r[10], r[11], lo, hi, 10);
            const u32 na = ld(SH_A + 32 * (t + 4) + lane), ne = ld(SH_E + 32 * (t + 4) + lane);
            fold(SH_K_BOOL_A + 32 * (t + 4) + lane, air_bool<F>(na));
            fold(SH_K_BOOL_E + 32 * (t + 4) + lane, air_bool<F>(ne));
            u32 nal, nah, nel, neh;
            pack(na, nal, nah); add3(nal, nah, r[6], r[7], r[8], r[9], r[10], r[11], 12);
            pack(ne, nel, neh); add2(nel, neh, r[6], r[7], al[0], ah[0], 14);
            if (lane < 16) fold(SH_K_ROUND + 16 * t + lane, mine);
#pragma unroll
            for (int j = 0; j < 3; j++) {
                A[j] = A[j + 1]; al[j] = al[j + 1]; ah[j] = ah[j + 1];
                E[j] = E[j + 1]; el[j] = el[j + 1]; eh[j] = eh[j + 1];
            }
            A[3] = na; al[3] = nal; ah[3] = nah;
            E[3] = ne; el[3] = nel; eh[3] = neh;
        }
        // finalization (k = SH_K_FINAL + 2 i): add2_expr_out(pack(h_out[i]), h_in[i], pack(a_chain[67 - i])), then e_chain for 4 + i
        mine = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const u32 x = ld(SH_H_OUT + 32 * j + lane);
            fold(SH_K_BOOL_OUT + 32 * j + lane, air_bool<F>(x));
            u32 lo, hi;
            pack(x, lo, hi);
            const int w = 3 - (j & 3);
            add2(lo, hi, bc(hin, 2 * j), bc(hin, 2 * j + 1), j < 4 ? al[w] : el[w], j < 4 ? ah[w] : eh[w], 2 * j);
        }
        if (lane < 16) fold(SH_K_FINAL + lane, mine);
        if constexpr (SHARDED) air_warp_store<F>(a, acc, i, lane, air_shard_odd(a, i));
        else air_warp_store<F>(a, acc, i, lane);
    }
}

// ---- host entry points ----------------------------------------------------------------------------------------------------
template <int F, bool WINDOW> static int32_t sh_generate(p3gpu_ctx *ctx, const u32 *d_inputs, size_t n, u32 *d_trace, const GenWindow &win) {
    sha256_air_generate_kernel<F, WINDOW><<<(unsigned)((n + SG_WARPS - 1) / SG_WARPS), 32 * SG_WARPS, 0, ctx->stream>>>(d_inputs, n, d_trace, win);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

static int32_t sh_check(int field, size_t n_hashes) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "SHA-256 AIR: unsupported field %d", field);
    P3_CHECK(n_hashes > 0 && (n_hashes & (n_hashes - 1)) == 0 && n_hashes <= ((size_t)1 << 32), P3GPU_EINVAL,
             "SHA-256 AIR: %zu hashes (need a power of two, at most 2^32)", n_hashes);
    return P3GPU_OK;
}

int32_t sha256_air_generate(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, u32 *d_trace) {
    P3_TRY(sh_check(field, n_hashes));
    const GenWindow win{};
    return field == BABY_BEAR ? sh_generate<BABY_BEAR, false>(ctx, d_inputs, n_hashes, d_trace, win)
                              : sh_generate<KOALA_BEAR, false>(ctx, d_inputs, n_hashes, d_trace, win);
}

int32_t sha256_air_generate_cols(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, size_t col0, size_t col1, u32 *d_out) {
    P3_TRY(sh_check(field, n_hashes));
    P3_TRY(air_check_window("SHA-256", col0, col1, SH_COLS));
    if (col0 == col1) return P3GPU_OK;
    const GenWindow win{col0, col1, 1};
    return field == BABY_BEAR ? sh_generate<BABY_BEAR, true>(ctx, d_inputs, n_hashes, d_out, win)
                              : sh_generate<KOALA_BEAR, true>(ctx, d_inputs, n_hashes, d_out, win);
}

int32_t sha256_air_quotient(p3gpu_ctx *ctx, int field, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q) {
    return air_hand_quotient(ctx, field, "SHA-256", (const void *)sha256_air_quotient_kernel<BABY_BEAR, false>,
                             (const void *)sha256_air_quotient_kernel<KOALA_BEAR, false>, SH_CONSTRAINTS, SQ_WARPS, SQ_SMEM, 0, d_lde, log_lde, log_n,
                             alpha, d_q);
}

int32_t sha256_air_quotient_sharded(p3gpu_ctx *ctx, int field, const AirHandShard &shard, const u32 *d_block, unsigned log_lde, unsigned log_n,
                                    const u32 *alpha, u32 *d_q) {
    const AirHandShard sh{shard.world, shard.rank, shard.col_starts, SH_COLS};
    return air_hand_quotient(ctx, field, "SHA-256", (const void *)sha256_air_quotient_kernel<BABY_BEAR, true>,
                             (const void *)sha256_air_quotient_kernel<KOALA_BEAR, true>, SH_CONSTRAINTS, SQ_WARPS, SQ_SMEM, 0, d_block, log_lde,
                             log_n, alpha, d_q, nullptr, 32, &sh);
}

}  // namespace p3
