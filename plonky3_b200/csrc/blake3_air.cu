// Blake3 AIR on the device: trace generation and quotient evaluation for the reference's Blake3Air (blake3-air/src), the AIR of
// `prove_prime_field_31 --objective blake-3-permutations` (examples/src/airs.rs), over BabyBear and KoalaBear.
//
//   trace generation   blake3-air/src/generation.rs:16-118: one compression per row, 9168 columns; row i hashes its 24 input words
//                      (16 message words, 8 chaining-value words) with counter i, block_len n (the row count), flags 0
//   constraints        blake3-air/src/air.rs:246-456 + air/src/utils.rs (add2, add3, xor_32_shift, pack_bits_le): 9632 constraints
//                      of degree <= 3 on the local row only, folded with alpha^(9631 - k) in eval order
//   quotient           uni-stark/src/prover.rs:462-827 over GENERATOR * K, |K| = 2 N (two quotient chunks), times 1 / Z_H
//
// Column layout (columns.rs Blake3Cols, repr(C)):
//   inputs [16][32] [0,512) | chaining_values [2][4][32] [512,768) | counter_low, counter_hi, block_len, flags [768,896) |
//   initial_row0 [4][2] [896,904) | initial_row2 [904,912) | full_rounds [7] [912,8528) | final_round_helpers [4][32] [8528,8656) |
//   outputs [4][4][32] [8656,9168)
// A FullRound is state_prime, state_middle, state_middle_prime, state_output; a state is row0 [4][2] 16-bit limbs (+0), row1 [4][32]
// bits (+8), row2 [4][2] limbs (+136), row3 [4][32] bits (+144), 272 columns.  Bits least significant first, limbs [lo, hi].
#include "common.h"
#include "air_program.cuh"

namespace p3 {

constexpr int B3_COLS = 9168, B3_CONSTRAINTS = 9632, B3_ROUNDS = 7;
constexpr int B3_CV = 512, B3_COUNTER = 768, B3_ROW0 = 896, B3_ROW2 = 904, B3_FULL = 912, B3_HELPERS = 8528, B3_OUT = 8656;
constexpr int B3_STATE = 272, B3_FULL_ROUND = 4 * B3_STATE;
constexpr int B3_S_ROW1 = 8, B3_S_ROW2 = 136, B3_S_ROW3 = 144;
// constraint indices: 896 booleans, 8 + 8 initial-row checks, 56 quarter rounds of 144, then the output checks
constexpr int B3_K_QR = 912, B3_QR = 144, B3_K_TAIL = B3_K_QR + 56 * B3_QR;

__constant__ u32 B3_IV[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au, 0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};
// message word of position i in round r: MSG_PERMUTATION applied r times (constants.rs permute between rounds)
__constant__ unsigned char B3_SCHEDULE[B3_ROUNDS][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15},  {2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8},
    {3, 4, 10, 12, 13, 2, 7, 14, 6, 5, 9, 0, 11, 15, 8, 1},  {10, 7, 12, 9, 14, 3, 13, 15, 4, 0, 11, 2, 5, 8, 1, 6},
    {12, 13, 9, 11, 15, 10, 14, 8, 7, 2, 5, 3, 0, 1, 6, 4},  {9, 14, 11, 5, 8, 12, 15, 1, 13, 3, 0, 10, 2, 6, 4, 7},
    {11, 15, 5, 0, 1, 9, 8, 6, 14, 10, 2, 12, 3, 4, 7, 13}};

__device__ __forceinline__ u32 b3_rotr(u32 v, int r) { return __funnelshift_r(v, v, r); }

// ---- trace generation -----------------------------------------------------------------------------------------------------
// One warp per row.  Every lane runs the whole compression in registers (the state and message words are warp-uniform, so the
// 16-word state, the 16 message words and the 8 chaining-value words are all compile-time indexed); lane l owns bit l of every
// 32-bit word.  A bit array is one 128-byte store per warp instruction (lane l writes column base + l); a state's eight limbs
// are written by lanes 0..7.  Nothing is read but the row's 96-byte input.
// WINDOW: only columns [win.col0, win.col1) are stored, as a dense n x (col1 - col0) matrix: the column block one rank of the sharded
// prover commits.  The whole compression still runs; only the stores are filtered.
constexpr int B3_GEN_WARPS = 8;

template <int F, bool WINDOW>
__global__ void __launch_bounds__(32 * B3_GEN_WARPS) blake3_air_generate_kernel(const u32 *inputs, size_t n, u32 *trace, const GenWindow win) {
    const unsigned lane = threadIdx.x & 31u;
    const size_t row = (size_t)blockIdx.x * B3_GEN_WARPS + (threadIdx.x >> 5);
    if (row >= n) return;
    const u32 ONE = Fp<F>::ONE;
    const u32 word = lane < 24 ? __ldg(inputs + row * 24 + lane) : 0u;
    u32 m[16], cv[8], v[16];
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = __shfl_sync(0xffffffffu, word, i);
#pragma unroll
    for (int i = 0; i < 8; i++) cv[i] = __shfl_sync(0xffffffffu, word, 16 + i);
    // the initial state: chaining value, IV[0..4], counter (low, high), block_len, flags
#pragma unroll
    for (int j = 0; j < 8; j++) v[j] = cv[j];
#pragma unroll
    for (int j = 0; j < 4; j++) v[8 + j] = B3_IV[j];
    v[12] = (u32)row; v[13] = (u32)(row >> 32); v[14] = (u32)n; v[15] = 0u;
    u32 *out = WINDOW ? trace + row * (win.col1 - win.col0) : trace + row * B3_COLS;
    auto put = [&](int c, u32 v) {
        if constexpr (WINDOW) {
            if ((size_t)c >= win.col0 && (size_t)c < win.col1) out[c - win.col0] = v;
        } else {
            out[c] = v;
        }
    };
    auto bits = [&](int col, u32 w) { put(col + lane, (w >> lane) & 1u ? ONE : 0u); };
    auto limbs = [&](int col, u32 w0, u32 w1, u32 w2, u32 w3) {             // [4][2] limbs: lane j < 8 writes limb j
        const unsigned j = lane >> 1;
        const u32 w = j == 0 ? w0 : j == 1 ? w1 : j == 2 ? w2 : w3;
        if (lane < 8) put(col + lane, to_monty<F>(lane & 1u ? w >> 16 : w & 0xffffu));
    };
    auto save = [&](int base) {                                             // generation.rs save_state_to_trace
        limbs(base, v[0], v[1], v[2], v[3]);
#pragma unroll
        for (int j = 0; j < 4; j++) bits(base + B3_S_ROW1 + 32 * j, v[4 + j]);
        limbs(base + B3_S_ROW2, v[8], v[9], v[10], v[11]);
#pragma unroll
        for (int j = 0; j < 4; j++) bits(base + B3_S_ROW3 + 32 * j, v[12 + j]);
    };
    // verifiable_half_round: (rot_1, rot_2) = (16, 12) for the first half, (8, 7) for the second
    auto half = [&](int a, int b, int c, int d, u32 mw, bool second) {
        v[a] = v[a] + v[b] + mw;
        v[d] = b3_rotr(v[d] ^ v[a], second ? 8 : 16);
        v[c] = v[c] + v[d];
        v[b] = b3_rotr(v[b] ^ v[c], second ? 7 : 12);
    };
#pragma unroll
    for (int w = 0; w < 16; w++) bits(32 * w, m[w]);
#pragma unroll
    for (int j = 0; j < 8; j++) bits(B3_CV + 32 * j, cv[j]);
#pragma unroll
    for (int j = 0; j < 4; j++) bits(B3_COUNTER + 32 * j, v[12 + j]);
    limbs(B3_ROW0, cv[0], cv[1], cv[2], cv[3]);
    limbs(B3_ROW2, B3_IV[0], B3_IV[1], B3_IV[2], B3_IV[3]);
#pragma unroll
    for (int r = 0; r < B3_ROUNDS; r++) {
        const int base = B3_FULL + B3_FULL_ROUND * r;
#pragma unroll
        for (int i = 0; i < 4; i++) half(i, 4 + i, 8 + i, 12 + i, m[2 * i], false);
        save(base);
#pragma unroll
        for (int i = 0; i < 4; i++) half(i, 4 + i, 8 + i, 12 + i, m[2 * i + 1], true);
        save(base + B3_STATE);
#pragma unroll
        for (int i = 0; i < 4; i++) half(i, 4 + (i + 1) % 4, 8 + (i + 2) % 4, 12 + (i + 3) % 4, m[8 + 2 * i], false);
        save(base + 2 * B3_STATE);
#pragma unroll
        for (int i = 0; i < 4; i++) half(i, 4 + (i + 1) % 4, 8 + (i + 2) % 4, 12 + (i + 3) % 4, m[9 + 2 * i], true);
        save(base + 3 * B3_STATE);
        const u32 t[16] = {m[2], m[6], m[3], m[10], m[7], m[0], m[4], m[13], m[1], m[11], m[12], m[5], m[9], m[14], m[15], m[8]};
#pragma unroll
        for (int i = 0; i < 16; i++) m[i] = t[i];                           // permute
    }
#pragma unroll
    for (int j = 0; j < 4; j++) {
        bits(B3_HELPERS + 32 * j, v[8 + j]);
        bits(B3_OUT + 32 * j, v[j] ^ v[8 + j]);
        bits(B3_OUT + 128 + 32 * j, v[4 + j] ^ v[12 + j]);
        bits(B3_OUT + 256 + 32 * j, v[8 + j] ^ cv[j]);
        bits(B3_OUT + 384 + 32 * j, v[12 + j] ^ cv[4 + j]);
    }
}

// ---- quotient -------------------------------------------------------------------------------------------------------------
// One warp per point of the quotient domain, persistent blocks of BQ_WARPS warps; the block holds the whole alpha-power table
// (alpha^(9631 - k), 154 KB) in shared memory, so rows are read from global memory as they are used, never staged: a 32-bit bit
// array is one coalesced 128-byte load (lane l reads bit l), a limb is a warp-uniform load.  Lane l owns bit l of every word:
//   - a boolean check of bit l is lane l's constraint;
//   - xor_32_shift(a, b, c, s): lane l forms xor(b[l], c[(l - s) mod 32]) with one shuffle, and a 16-bit pack sums the weighted
//     bits over a half warp (four shuffles), then both halves are broadcast;
//   - the 16 limb-level constraints of a quarter round (add3 / add2 / pack checks, two each) are warp-uniform values; lane j < 16
//     keeps the j-th and folds it.
// Each lane folds its constraints with air_qmac; the warp adds the 32 partial sums and multiplies by 1 / Z_H.
// SHARDED: one rank's chunk-major row block (AirHandQArgs); every column address goes through the unit table behind the alpha
// powers (air_program.cuh AirShardRow), the block's rows are the points, and the quotient lands in the block's slice.
constexpr int BQ_WARPS = 16;
constexpr size_t BQ_SMEM = (size_t)B3_CONSTRAINTS * 16;

// a Blake3State's four column bases: row0[j] limbs at r0 + 2j, row1[j] bits at r1 + 32j, row2[j] at r2 + 2j, row3[j] at r3 + 32j
struct B3View { int r0, r1, r2, r3; };
__device__ __forceinline__ B3View b3_state(int base) { return {base, base + B3_S_ROW1, base + B3_S_ROW2, base + B3_S_ROW3}; }

template <int F, bool SHARDED> __global__ void __launch_bounds__(32 * BQ_WARPS, 1) blake3_air_quotient_kernel(const AirHandQArgs a) {
    extern __shared__ uint4 bq_sm[];
    const uint4 *ap = bq_sm;
    u64 *units = reinterpret_cast<u64 *>(bq_sm + B3_CONSTRAINTS);
    for (int t = threadIdx.x; t < B3_CONSTRAINTS; t += blockDim.x) bq_sm[t] = __ldg(a.apow + t);
    if constexpr (SHARDED) air_shard_table_load(a, units);
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const u32 n_pts = SHARDED ? a.rows : 1u << a.d.log_q;
    const u32 T16 = to_monty<F>(1u << 16), T17 = fp_double<F>(T16), T32 = mont_mul<F>(T16, T16), T33 = fp_double<F>(T32);
    const u32 wpow = to_monty<F>(1u << (lane & 15u));                  // weight of this lane's bit in its 16-bit limb
    auto add = [](u32 x, u32 y) { return fp_add<F>(x, y); };
    auto sub = [](u32 x, u32 y) { return fp_sub<F>(x, y); };
    auto mul = [](u32 x, u32 y) { return mont_mul<F>(x, y); };
    // pack_bits_le of the lane-distributed bits v over [0, 16) and [16, 32): (lo, hi), warp-uniform
    auto pack = [&](u32 v, u32 &lo, u32 &hi) {
        u32 s = mul(v, wpow);
#pragma unroll
        for (int o = 8; o; o >>= 1) s = add(s, __shfl_xor_sync(0xffffffffu, s, o));
        lo = __shfl_sync(0xffffffffu, s, 0); hi = __shfl_sync(0xffffffffu, s, 16);
    };
    for (u32 i = blockIdx.x * BQ_WARPS + warp; i < n_pts; i += gridDim.x * BQ_WARPS) {
        const u32 *row = SHARDED ? a.lde : a.lde + (size_t)air_bitrev(i, a.d.log_q) * B3_COLS;
        const AirShardRow sr{a.lde, units, i};
        auto ld = [row, sr](int c) {
            if constexpr (SHARDED) return sr.ld((u32)c);
            else return __ldg(row + c);
        };
        u64 acc[4] = {0, 0, 0, 0};
        auto fold = [&](int k, u32 c) { air_qmac<F>(acc, c, ap[k]); };
        // the initialisation inputs are boolean (k 0..895: column k)
        for (int c = lane; c < B3_ROW0; c += 32) fold(c, air_bool<F>(ld(c)));
        // initial row0 = packed chaining_values[0] (k 896..903), initial row2 = IV (k 904..911)
        {
            u32 mine = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                u32 lo, hi;
                pack(ld(B3_CV + 32 * j + lane), lo, hi);
                if (lane == 2 * j) mine = sub(lo, ld(B3_ROW0 + 2 * j));
                if (lane == 2 * j + 1) mine = sub(hi, ld(B3_ROW0 + 2 * j + 1));
            }
            if (lane >= 8 && lane < 16) {
                const unsigned j = (lane - 8) >> 1;
                const u32 ivj = j == 0 ? B3_IV[0] : j == 1 ? B3_IV[1] : j == 2 ? B3_IV[2] : B3_IV[3];
                mine = sub(ld(B3_ROW2 + lane - 8), to_monty<F>(lane & 1u ? ivj >> 16 : ivj & 0xffffu));
            }
            if (lane < 16) fold(896 + lane, mine);
        }
        // message limbs: lane l holds limb (l & 1) of message word l >> 1
        u32 mlimb = 0;
#pragma unroll 4
        for (int w = 0; w < 16; w++) {
            u32 lo, hi;
            pack(ld(32 * w + lane), lo, hi);
            if ((lane >> 1) == (unsigned)w) mlimb = lane & 1u ? hi : lo;
        }
        // 7 rounds x (4 column + 4 diagonal) quarter rounds, 144 constraints each (air.rs quarter_round_function):
        //   add3 (0, 1) | xor_32_shift(a', d, d', 16) (2..35) | add2 (36, 37) | xor_32_shift(c', b, b', 12) (38..71) |
        //   add3 (72, 73) | xor_32_shift(a'', d', d'', 8) (74..107) | add2 (108, 109) | xor_32_shift(c'', b', b'', 7) (110..143)
        B3View in = {B3_ROW0, B3_CV + 128, B3_ROW2, B3_COUNTER};
#pragma unroll 1
        for (int r = 0; r < B3_ROUNDS; r++) {
            const int base = B3_FULL + B3_FULL_ROUND * r;
            const B3View sp = b3_state(base), sm = b3_state(base + B3_STATE), smp = b3_state(base + 2 * B3_STATE),
                         so = b3_state(base + 3 * B3_STATE);
#pragma unroll 1
            for (int qr = 0; qr < 8; qr++) {
                const bool diag = qr >= 4;
                const int x = qr & 3, j1 = diag ? (x + 1) & 3 : x, j2 = diag ? (x + 2) & 3 : x, j3 = diag ? (x + 3) & 3 : x;
                const B3View s0 = diag ? sm : in, s1 = diag ? smp : sp, s2 = diag ? so : sm;
                const int k = B3_K_QR + B3_QR * (8 * r + qr);
                const int mi0 = B3_SCHEDULE[r][2 * qr], mi1 = B3_SCHEDULE[r][2 * qr + 1];  // m_vector[2i (+ 8)], [2i + 1 (+ 8)]
                const u32 m0l = __shfl_sync(0xffffffffu, mlimb, 2 * mi0), m0h = __shfl_sync(0xffffffffu, mlimb, 2 * mi0 + 1);
                const u32 m1l = __shfl_sync(0xffffffffu, mlimb, 2 * mi1), m1h = __shfl_sync(0xffffffffu, mlimb, 2 * mi1 + 1);
                // limbs a, c (input), a', c' (half-way), a'', c'' (output); bits b, d, b', d', b'', d'' of this lane
                const u32 a0 = ld(s0.r0 + 2 * x), a1 = ld(s0.r0 + 2 * x + 1), c0 = ld(s0.r2 + 2 * j2), c1 = ld(s0.r2 + 2 * j2 + 1);
                const u32 ap0 = ld(s1.r0 + 2 * x), ap1 = ld(s1.r0 + 2 * x + 1), cp0 = ld(s1.r2 + 2 * j2), cp1 = ld(s1.r2 + 2 * j2 + 1);
                const u32 ao0 = ld(s2.r0 + 2 * x), ao1 = ld(s2.r0 + 2 * x + 1), co0 = ld(s2.r2 + 2 * j2), co1 = ld(s2.r2 + 2 * j2 + 1);
                const u32 b = ld(s0.r1 + 32 * j1 + lane), d = ld(s0.r3 + 32 * j3 + lane);
                const u32 bp = ld(s1.r1 + 32 * j1 + lane), dp = ld(s1.r3 + 32 * j3 + lane);
                const u32 bo = ld(s2.r1 + 32 * j1 + lane), dout = ld(s2.r3 + 32 * j3 + lane);
                // booleans of d', b', d'', b'' (the c argument of each xor_32_shift)
                fold(k + 2 + lane, air_bool<F>(dp)); fold(k + 38 + lane, air_bool<F>(bp)); fold(k + 74 + lane, air_bool<F>(dout)); fold(k + 110 + lane, air_bool<F>(bo));
                u32 lo, hi, mine = 0;
                // add3(a', a, pack(b), m0): acc (acc + 2^32) (acc + 2 2^32), acc16 (acc16 + 2^16) (acc16 + 2 2^16)
                auto add3 = [&](u32 x0, u32 x1, u32 y0, u32 y1, u32 l, u32 h, u32 z0, u32 z1, int j) {
                    const u32 acc16 = sub(sub(sub(x0, y0), l), z0), acc32 = sub(sub(sub(x1, y1), h), z1);
                    const u32 accv = add(acc16, mul(acc32, T16));
                    if (lane == (unsigned)j) mine = mul(mul(accv, add(accv, T32)), add(accv, T33));
                    if (lane == (unsigned)j + 1) mine = mul(mul(acc16, add(acc16, T16)), add(acc16, T17));
                };
                auto add2 = [&](u32 x0, u32 x1, u32 y0, u32 y1, u32 l, u32 h, int j) {
                    const u32 acc16 = sub(sub(x0, y0), l), acc32 = sub(sub(x1, y1), h);
                    const u32 accv = add(acc16, mul(acc32, T16));
                    if (lane == (unsigned)j) mine = mul(accv, add(accv, T32));
                    if (lane == (unsigned)j + 1) mine = mul(acc16, add(acc16, T16));
                };
                // xor_32_shift(x, bb, cc, s): x[0] - pack(lo), x[1] - pack(hi) of xor(bb[l], cc[(l - s) mod 32])
                auto xsh = [&](u32 x0, u32 x1, u32 bb, u32 cc, int s, int j) {
                    pack(air_bxor<F>(bb, __shfl_sync(0xffffffffu, cc, (lane - s) & 31u)), lo, hi);
                    if (lane == (unsigned)j) mine = sub(x0, lo);
                    if (lane == (unsigned)j + 1) mine = sub(x1, hi);
                };
                pack(b, lo, hi);    add3(ap0, ap1, a0, a1, lo, hi, m0l, m0h, 0);
                xsh(ap0, ap1, d, dp, 16, 2);
                pack(dp, lo, hi);   add2(cp0, cp1, c0, c1, lo, hi, 4);
                xsh(cp0, cp1, b, bp, 12, 6);
                pack(bp, lo, hi);   add3(ao0, ao1, ap0, ap1, lo, hi, m1l, m1h, 8);
                xsh(ao0, ao1, dp, dout, 8, 10);
                pack(dout, lo, hi); add2(co0, co1, cp0, cp1, lo, hi, 12);
                xsh(co0, co1, bp, bo, 7, 14);
                // lane j < 16 folds the j-th limb-level constraint: pair p = j >> 1 sits at 36 (p >> 1) + 34 (p & 1)
                if (lane < 16) fold(k + 36 * (lane >> 2) + 34 * ((lane >> 1) & 1u) + (lane & 1u), mine);
            }
            in = so;
        }
        // final xors (air.rs:384-455), state = full_rounds[6].state_output
        {
            const B3View so = b3_state(B3_FULL + B3_FULL_ROUND * 6 + 3 * B3_STATE);
            const int k = B3_K_TAIL;
            u32 mine = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const u32 h = ld(B3_HELPERS + 32 * j + lane), o0 = ld(B3_OUT + 32 * j + lane);
                const u32 o1 = ld(B3_OUT + 128 + 32 * j + lane), o2 = ld(B3_OUT + 256 + 32 * j + lane), o3 = ld(B3_OUT + 384 + 32 * j + lane);
                const u32 r1 = ld(so.r1 + 32 * j + lane), r3 = ld(so.r3 + 32 * j + lane);
                const u32 cv0 = ld(B3_CV + 32 * j + lane), cv1 = ld(B3_CV + 128 + 32 * j + lane);
                u32 lo, hi;
                // helpers pack to state_output.row2 (k + 0..7)
                pack(h, lo, hi);
                if (lane == 2 * j) mine = sub(lo, ld(so.r2 + 2 * j));
                if (lane == 2 * j + 1) mine = sub(hi, ld(so.r2 + 2 * j + 1));
                // outputs[0] booleans (k + 8 .. 135)
                fold(k + 8 + 32 * j + lane, air_bool<F>(o0));
                // xor_32_shift(row0[j], outputs[0][j], helpers[j], 0): 32 booleans of helpers[j], then two packs (k + 136 + 34 j ..)
                fold(k + 136 + 34 * j + lane, air_bool<F>(h));
                pack(air_bxor<F>(o0, h), lo, hi);
                if (lane == 16 + 2 * j) mine = sub(ld(so.r0 + 2 * j), lo);
                if (lane == 17 + 2 * j) mine = sub(ld(so.r0 + 2 * j + 1), hi);
                // outputs[1] = row1 ^ row3, outputs[2] = chaining_values[0] ^ helpers, outputs[3] = chaining_values[1] ^ row3 (k + 272 ..)
                fold(k + 272 + 32 * j + lane, sub(o1, air_bxor<F>(r1, r3)));
                fold(k + 400 + 32 * j + lane, sub(o2, air_bxor<F>(cv0, h)));
                fold(k + 528 + 32 * j + lane, sub(o3, air_bxor<F>(cv1, r3)));
            }
            if (lane < 8) fold(k + lane, mine);
            else if (lane >= 16 && lane < 24) fold(k + 136 + 34 * ((lane - 16) >> 1) + 32 + (lane & 1u), mine);
        }
        if constexpr (SHARDED) air_warp_store<F>(a, acc, i, lane, air_shard_odd(a, i));
        else air_warp_store<F>(a, acc, i, lane);
    }
}

// ---- host entry points ----------------------------------------------------------------------------------------------------
template <int F, bool WINDOW> static int32_t b3_generate(p3gpu_ctx *ctx, const u32 *d_inputs, size_t n, u32 *d_trace, const GenWindow &win) {
    blake3_air_generate_kernel<F, WINDOW><<<(unsigned)((n + B3_GEN_WARPS - 1) / B3_GEN_WARPS), 32 * B3_GEN_WARPS, 0, ctx->stream>>>(d_inputs, n,
                                                                                                                             d_trace, win);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

static int32_t b3_check(int field, size_t n_hashes) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "Blake3 AIR: unsupported field %d", field);
    P3_CHECK(n_hashes > 0 && (n_hashes & (n_hashes - 1)) == 0 && n_hashes <= ((size_t)1 << 32), P3GPU_EINVAL,
             "Blake3 AIR: %zu hashes (need a power of two, at most 2^32)", n_hashes);
    return P3GPU_OK;
}

int32_t blake3_air_generate(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, u32 *d_trace) {
    P3_TRY(b3_check(field, n_hashes));
    const GenWindow win{};
    return field == BABY_BEAR ? b3_generate<BABY_BEAR, false>(ctx, d_inputs, n_hashes, d_trace, win)
                              : b3_generate<KOALA_BEAR, false>(ctx, d_inputs, n_hashes, d_trace, win);
}

int32_t blake3_air_generate_cols(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, size_t col0, size_t col1, u32 *d_out) {
    P3_TRY(b3_check(field, n_hashes));
    P3_TRY(air_check_window("Blake3", col0, col1, B3_COLS));
    if (col0 == col1) return P3GPU_OK;
    const GenWindow win{col0, col1, 1};
    return field == BABY_BEAR ? b3_generate<BABY_BEAR, true>(ctx, d_inputs, n_hashes, d_out, win)
                              : b3_generate<KOALA_BEAR, true>(ctx, d_inputs, n_hashes, d_out, win);
}

int32_t blake3_air_quotient(p3gpu_ctx *ctx, int field, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q) {
    return air_hand_quotient(ctx, field, "Blake3", (const void *)blake3_air_quotient_kernel<BABY_BEAR, false>,
                             (const void *)blake3_air_quotient_kernel<KOALA_BEAR, false>, B3_CONSTRAINTS, BQ_WARPS, BQ_SMEM, 0, d_lde, log_lde, log_n,
                             alpha, d_q);
}

int32_t blake3_air_quotient_sharded(p3gpu_ctx *ctx, int field, const AirHandShard &shard, const u32 *d_block, unsigned log_lde, unsigned log_n,
                                    const u32 *alpha, u32 *d_q) {
    const AirHandShard sh{shard.world, shard.rank, shard.col_starts, B3_COLS};
    return air_hand_quotient(ctx, field, "Blake3", (const void *)blake3_air_quotient_kernel<BABY_BEAR, true>,
                             (const void *)blake3_air_quotient_kernel<KOALA_BEAR, true>, B3_CONSTRAINTS, BQ_WARPS, BQ_SMEM, 0, d_block, log_lde,
                             log_n, alpha, d_q, nullptr, 32, &sh);
}

}  // namespace p3
