// Keccak-f AIR on the device: trace generation and quotient evaluation for the reference's KeccakAir (keccak-air/src), the AIR of
// `prove_prime_field_31 --objective keccak-f-permutations` (examples/src/airs.rs), over BabyBear and KoalaBear.
//
//   trace generation   keccak-air/src/generation.rs:16-161: one Keccak round per row, 24 rows per permutation, 2633 columns;
//                      height (24 n).next_power_of_two(), padding = the zero-input permutation's rows repeated, the last copy cut
//   constraints        keccak-air/src/air.rs:44-205 + round_flags.rs:21-48: 3182 constraints of degree <= 3, folded with
//                      alpha^(3181 - k) in eval order (the first asserted constraint gets the highest power, uni-stark/src/folder.rs)
//   quotient           uni-stark/src/prover.rs:462-827 over GENERATOR * K, |K| = 2 N (two quotient chunks), times 1 / Z_H
//
// Column layout (columns.rs KeccakCols, repr(C)):
//   step_flags [0,24) | export 24 | preimage [25,125) | a [125,225) | c [225,545) | c_prime [545,865) | a_prime [865,2465) |
//   a_prime_prime [2465,2565) | a_prime_prime_0_0_bits [2565,2629) | a_prime_prime_prime_0_0_limbs [2629,2633)
// preimage, a, a_prime, a_prime_prime are stored [y][x]; limbs are 16 bits, four per u64, least significant first.
#include "common.h"
#include "air_program.cuh"

namespace p3 {

constexpr int KA_COLS = 2633, KA_ROUNDS = 24, KA_NEXT_COLS = 225, KA_CONSTRAINTS = 3182;
constexpr int KA_STEP = 0, KA_EXPORT = 24, KA_PRE = 25, KA_A = 125, KA_C = 225, KA_CP = 545, KA_AP = 865, KA_APP = 2465, KA_APP_BITS = 2565,
              KA_APPP = 2629;

// constants.rs: rotation offsets R[x][y] and round constants RC[r] (FIPS 202 rho and iota)
__constant__ unsigned char KA_R[5][5] = {
    {0, 36, 3, 41, 18}, {1, 44, 10, 45, 2}, {62, 6, 43, 15, 61}, {28, 55, 25, 21, 56}, {27, 20, 39, 8, 14}};
__constant__ u64 KA_RC[24] = {
    0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808Aull, 0x8000000080008000ull, 0x000000000000808Bull, 0x0000000080000001ull,
    0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008Aull, 0x0000000000000088ull, 0x0000000080008009ull, 0x000000008000000Aull,
    0x000000008000808Bull, 0x800000000000008Bull, 0x8000000000008089ull, 0x8000000000008003ull, 0x8000000000008002ull, 0x8000000000000080ull,
    0x000000000000800Aull, 0x800000008000000Aull, 0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull};

__device__ __forceinline__ u64 ka_rotl(u64 v, unsigned r) { return r ? (v << r) | (v >> (64 - r)) : v; }

// ---- trace generation -----------------------------------------------------------------------------------------------------
// One warp per 24-row block (one permutation).  Lanes 0..24 run the round on the state words in shared memory (index x + 5 y);
// then the whole warp writes the round's row in column order, consecutive lanes on consecutive words: every store instruction
// is one contiguous 128-byte span.  Rows are 2633 words (odd), so only 4-byte stores line up with every row.
// Blocks >= n_real are padding: a copy of the zero-input block `zero` (24 x 2633 words), which a first launch (n_real = 1, no
// inputs) computes once, cut at the trace height.
struct KaState { u64 in[25], a[25], c[5], cp[5], ap[25], app[25]; };
constexpr int KA_GEN_WARPS = 4;

template <int F>
__global__ void __launch_bounds__(32 * KA_GEN_WARPS) keccak_air_generate_kernel(const u64 *inputs, size_t n_real, size_t height, u32 *trace,
                                                                                const u32 *zero) {
    __shared__ KaState sts[KA_GEN_WARPS];
    KaState &s = sts[threadIdx.x >> 5];
    const unsigned lane = threadIdx.x & 31u;
    const size_t blk = (size_t)blockIdx.x * KA_GEN_WARPS + (threadIdx.x >> 5);
    const size_t row0 = blk * KA_ROUNDS;
    if (row0 >= height) return;
    const size_t rows = min((size_t)KA_ROUNDS, height - row0);
    u32 *out = trace + row0 * KA_COLS;
    if (blk >= n_real) {                                         // padding: the zero-input block, truncated
        const size_t words = rows * KA_COLS;
        for (size_t w = lane; w < words; w += 32) out[w] = __ldg(zero + w);
        return;
    }
    if (lane < 25) {
        const u64 v = inputs ? __ldg(inputs + blk * 25 + lane) : 0ull;    // input[x + 5 y] = state[x][y]
        s.in[lane] = v; s.a[lane] = v;
    }
    __syncwarp();
    const u32 ONE = Fp<F>::ONE;
    auto limb = [](u64 v, int l) { return to_monty<F>((u32)(v >> (16 * l)) & 0xffffu); };
    for (int r = 0; r < (int)rows; r++) {
        const unsigned x = lane % 5, y = lane / 5;
        if (lane < 5) s.c[x] = s.a[x] ^ s.a[x + 5] ^ s.a[x + 10] ^ s.a[x + 15] ^ s.a[x + 20];
        __syncwarp();
        if (lane < 5) s.cp[x] = s.c[x] ^ s.c[(x + 4) % 5] ^ ka_rotl(s.c[(x + 1) % 5], 1);
        __syncwarp();
        if (lane < 25) s.ap[lane] = s.a[lane] ^ s.c[x] ^ s.cp[x];
        __syncwarp();
        if (lane < 25) {
            // B[x][y] = ROT(A'[(x + 3y) % 5][x], R[(x + 3y) % 5][x]);  A''[x][y] = B[x][y] ^ (~B[x+1][y] & B[x+2][y])
            auto b = [&](unsigned bx) { const unsigned ax = (bx + 3 * y) % 5; return ka_rotl(s.ap[ax + 5 * bx], KA_R[ax][bx]); };
            s.app[lane] = b(x) ^ (~b((x + 1) % 5) & b((x + 2) % 5));
        }
        __syncwarp();
        const u64 appp = s.app[0] ^ KA_RC[r];
        u32 *row = out + (size_t)r * KA_COLS;
        for (int col = lane; col < KA_COLS; col += 32) {
            u32 v;
            if (col < KA_EXPORT) v = col == r ? ONE : 0u;
            else if (col < KA_PRE) v = 0u;                                   // export: never set by generate_trace_rows
            else if (col < KA_A) v = limb(s.in[(col - KA_PRE) >> 2], (col - KA_PRE) & 3);
            else if (col < KA_C) v = limb(s.a[(col - KA_A) >> 2], (col - KA_A) & 3);
            else if (col < KA_CP) v = (s.c[(col - KA_C) >> 6] >> ((col - KA_C) & 63)) & 1 ? ONE : 0u;
            else if (col < KA_AP) v = (s.cp[(col - KA_CP) >> 6] >> ((col - KA_CP) & 63)) & 1 ? ONE : 0u;
            else if (col < KA_APP) v = (s.ap[(col - KA_AP) >> 6] >> ((col - KA_AP) & 63)) & 1 ? ONE : 0u;
            else if (col < KA_APP_BITS) v = limb(s.app[(col - KA_APP) >> 2], (col - KA_APP) & 3);
            else if (col < KA_APPP) v = (s.app[0] >> (col - KA_APP_BITS)) & 1 ? ONE : 0u;
            else v = limb(appp, col - KA_APPP);
            row[col] = v;
        }
        __syncwarp();
        if (lane < 25) s.a[lane] = lane == 0 ? appp : s.app[lane];         // this round's output is the next round's input
        __syncwarp();
    }
}

// ---- quotient -------------------------------------------------------------------------------------------------------------
// One warp per point of the quotient domain, persistent blocks of KQ_WARPS warps.  The warp stages its local row (2633 words)
// and the 225 next-row words the constraints read into shared memory with 4-byte cp.async (rows are only 4-byte aligned), then
// its lanes evaluate disjoint constraint subsets: lane l owns bit positions z = l and l + 32 of every 64-bit word; a 16-bit limb
// check sums its 16 weighted bits over a half warp with four shuffles; the flag, preimage and output-transition checks are
// spread over the lanes by index.  Each lane folds its constraints with alpha^(3181 - k) from the block's shared table (51 KB),
// the warp adds the 32 partial sums and multiplies by 1 / Z_H.  The next row of point i is the local row of point i + 2, which
// the warp two places on is loading at the same time: it comes from L2.
constexpr int KQ_WARPS = 12;
constexpr int KQ_ROW = KA_COLS + KA_NEXT_COLS;                       // staged words per warp
constexpr size_t KQ_SMEM = (size_t)KA_CONSTRAINTS * 16 + (size_t)KQ_WARPS * KQ_ROW * 4;

__device__ __forceinline__ void ka_cp_async4(u32 *dst, const u32 *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}

template <int F> __global__ void __launch_bounds__(32 * KQ_WARPS, 1) keccak_air_quotient_kernel(const AirHandQArgs a) {
    extern __shared__ uint4 kq_sm[];
    const uint4 *ap = kq_sm;
    for (int t = threadIdx.x; t < KA_CONSTRAINTS; t += blockDim.x) kq_sm[t] = __ldg(a.apow + t);
    __syncthreads();
    const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    u32 *L = reinterpret_cast<u32 *>(kq_sm + KA_CONSTRAINTS) + (size_t)warp * KQ_ROW;
    const u32 *N = L + KA_COLS;
    const u32 n_pts = 1u << a.d.log_q, mask = n_pts - 1u;
    const u32 ONE = Fp<F>::ONE, TWO = fp_double<F>(ONE), FOUR = fp_double<F>(TWO);
    const u32 wpow = to_monty<F>(1u << (lane & 15u));                // weight of this lane's bits in their limb
    auto add = [](u32 x, u32 y) { return fp_add<F>(x, y); };
    auto sub = [](u32 x, u32 y) { return fp_sub<F>(x, y); };
    auto mul = [](u32 x, u32 y) { return mont_mul<F>(x, y); };
    // (sum of this half warp's weighted v0, of its weighted v1): the limbs (lane / 16) and 2 + (lane / 16) of a 64-bit word
    auto limbs = [&](u32 v0, u32 v1, u32 &s0, u32 &s1) {
        s0 = mul(v0, wpow); s1 = mul(v1, wpow);
#pragma unroll
        for (int o = 8; o; o >>= 1) { s0 = add(s0, __shfl_xor_sync(0xffffffffu, s0, o)); s1 = add(s1, __shfl_xor_sync(0xffffffffu, s1, o)); }
    };
    const unsigned z0 = lane, z1 = lane + 32, hl = lane >> 4;          // lane's bit positions; its limbs are hl and 2 + hl
    for (u32 i = blockIdx.x * KQ_WARPS + warp; i < n_pts; i += gridDim.x * KQ_WARPS) {
        const u32 m = air_bitrev(i, a.d.log_q), mn = air_bitrev((i + 2u) & mask, a.d.log_q);
        {
            const u32 *row = a.lde + (size_t)m * KA_COLS, *nrow = a.lde + (size_t)mn * KA_COLS;
            __syncwarp();                                           // the previous point's reads are done
            for (int c = lane; c < KA_COLS; c += 32) ka_cp_async4(L + c, row + c);
            for (int c = lane; c < KA_NEXT_COLS; c += 32) ka_cp_async4(L + KA_COLS + c, nrow + c);
            asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
            __syncwarp();
        }
        u32 first, last, trans;
        air_selectors<F>(a.d, i, (i & 1u) ? a.zh[1] : a.zh[0], first, last, trans);
        const u32 nf = sub(ONE, L[KA_STEP + 23]), tnf = mul(trans, nf), f0 = L[KA_STEP];
        u64 acc[4] = {0, 0, 0, 0};
        auto fold = [&](int k, u32 c) { air_qmac<F>(acc, c, ap[k]); };
        // round flags (round_flags.rs:32-47): k 0..47
        for (int k = lane; k < 48; k += 32) {
            u32 c;
            if (k == 0) c = mul(first, sub(L[0], ONE));
            else if (k < 24) c = mul(first, L[k]);
            else c = mul(trans, sub(L[k - 24], N[(k - 23) % 24]));
            fold(k, c);
        }
        // first step: preimage = a (k 48..147); transition and not final: preimage = next preimage (k 148..247), y-outer
        for (int j = lane; j < 200; j += 32) {
            const u32 c = j < 100 ? mul(f0, sub(L[KA_PRE + j], L[KA_A + j])) : mul(tnf, sub(L[KA_PRE + j - 100], N[KA_PRE + j - 100]));
            fold(48 + j, c);
        }
        // export is boolean (248) and zero unless final step (249)
        if (lane < 2) fold(248 + lane, lane == 0 ? air_bool<F>(L[KA_EXPORT]) : mul(nf, L[KA_EXPORT]));
        // per x: 64 c bools, then 64 c' = xor3(c[x][z], c[x-1][z], c[x+1][z-1]) (k 250..889)
#pragma unroll 1
        for (int x = 0; x < 5; x++) {
            const u32 *c = L + KA_C + 64 * x, *cm = L + KA_C + 64 * ((x + 4) % 5), *cq = L + KA_C + 64 * ((x + 1) % 5), *cp = L + KA_CP + 64 * x;
            const int k = 250 + 128 * x;
            fold(k + z0, air_bool<F>(c[z0])); fold(k + z1, air_bool<F>(c[z1]));
            fold(k + 64 + z0, sub(cp[z0], air_bxor<F>(air_bxor<F>(c[z0], cm[z0]), cq[(z0 + 63) & 63])));
            fold(k + 64 + z1, sub(cp[z1], air_bxor<F>(air_bxor<F>(c[z1], cm[z1]), cq[(z1 + 63) & 63])));
        }
        // x-outer, y-inner: 64 a' bools, then a[y][x] limb = sum 2^z xor(a'[y][x][z], xor(c[x][z], c'[x][z])) (k 890..2589)
#pragma unroll 1
        for (int x = 0; x < 5; x++) {
            const u32 cc0 = air_bxor<F>(L[KA_C + 64 * x + z0], L[KA_CP + 64 * x + z0]), cc1 = air_bxor<F>(L[KA_C + 64 * x + z1], L[KA_CP + 64 * x + z1]);
#pragma unroll 1
            for (int y = 0; y < 5; y++) {
                const u32 *apx = L + KA_AP + 64 * (5 * y + x);
                const int k = 890 + 68 * (5 * x + y);
                fold(k + z0, air_bool<F>(apx[z0])); fold(k + z1, air_bool<F>(apx[z1]));
                u32 s0, s1;
                limbs(air_bxor<F>(apx[z0], cc0), air_bxor<F>(apx[z1], cc1), s0, s1);
                const u32 *al = L + KA_A + 4 * (5 * y + x);
                if ((lane & 15u) == 0) fold(k + 64 + hl, sub(s0, al[hl]));
                else if ((lane & 15u) == 1) fold(k + 66 + hl, sub(s1, al[2 + hl]));
            }
        }
        // parity: diff = sum_y a'[y][x][z] - c'[x][z], diff (diff - 2) (diff - 4) (k 2590..2909)
#pragma unroll 1
        for (int x = 0; x < 5; x++) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const unsigned z = h ? z1 : z0;
                u32 sum = L[KA_AP + 64 * x + z];
#pragma unroll
                for (int y = 1; y < 5; y++) sum = add(sum, L[KA_AP + 64 * (5 * y + x) + z]);
                const u32 diff = sub(sum, L[KA_CP + 64 * x + z]);
                fold(2590 + 64 * x + z, mul(mul(diff, sub(diff, TWO)), sub(diff, FOUR)));
            }
        }
        // chi, y-outer: a''[y][x] limb = sum 2^z xor(andn(B[x+1][y][z], B[x+2][y][z]), B[x][y][z]) (k 2910..3009)
#pragma unroll 1
        for (int y = 0; y < 5; y++) {
#pragma unroll 1
            for (int x = 0; x < 5; x++) {
                u32 v[2];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const unsigned z = h ? z1 : z0;
                    // B[bx][y][z] = a'[bx][(bx + 3y) % 5][(z - R) mod 64] (columns.rs b())
                    auto b = [&](int bx) { const int ax = (bx + 3 * y) % 5; return L[KA_AP + 64 * (5 * bx + ax) + ((z + 64 - KA_R[ax][bx]) & 63)]; };
                    const u32 andn = mul(sub(ONE, b((x + 1) % 5)), b((x + 2) % 5));
                    v[h] = air_bxor<F>(andn, b(x));
                }
                u32 s0, s1;
                limbs(v[0], v[1], s0, s1);
                const u32 *al = L + KA_APP + 4 * (5 * y + x);
                const int k = 2910 + 4 * (5 * y + x);
                if ((lane & 15u) == 0) fold(k + hl, sub(s0, al[hl]));
                else if ((lane & 15u) == 1) fold(k + 2 + hl, sub(s1, al[2 + hl]));
            }
        }
        // a''[0,0] bits: bools (k 3010..3073), their limbs = a''[0][0] (3074..3077), iota: limbs of xor(rc bit, bit) = a''' (3078..3081)
        {
            const u32 b0 = L[KA_APP_BITS + z0], b1 = L[KA_APP_BITS + z1];
            fold(3010 + z0, air_bool<F>(b0)); fold(3010 + z1, air_bool<F>(b1));
            u32 s0, s1;
            limbs(b0, b1, s0, s1);
            if ((lane & 15u) == 0) fold(3074 + hl, sub(s0, L[KA_APP + hl]));
            else if ((lane & 15u) == 1) fold(3076 + hl, sub(s1, L[KA_APP + 2 + hl]));
            u32 rc0 = 0, rc1 = 0;                                   // sum of the step flags of the rounds whose RC has bit z
#pragma unroll 4
            for (int r = 0; r < KA_ROUNDS; r++) {
                const u64 rc = KA_RC[r];
                if ((rc >> z0) & 1) rc0 = add(rc0, L[KA_STEP + r]);
                if ((rc >> z1) & 1) rc1 = add(rc1, L[KA_STEP + r]);
            }
            limbs(air_bxor<F>(rc0, b0), air_bxor<F>(rc1, b1), s0, s1);
            if ((lane & 15u) == 0) fold(3078 + hl, sub(s0, L[KA_APPP + hl]));
            else if ((lane & 15u) == 1) fold(3080 + hl, sub(s1, L[KA_APPP + 2 + hl]));
        }
        // transition and not final: a'''[y][x] = next a[y][x], x-outer, y-inner (k 3082..3181)
        for (int j = lane; j < 100; j += 32) {
            const int x = j / 20, y = (j / 4) % 5, l = j & 3, yx = 5 * y + x;
            const u32 out = yx == 0 ? L[KA_APPP + l] : L[KA_APP + 4 * yx + l];
            fold(3082 + j, mul(tnf, sub(out, N[KA_A + 4 * yx + l])));
        }
        air_warp_store<F>(a, acc, i, lane);
    }
}

// ---- host entry points ----------------------------------------------------------------------------------------------------
size_t keccak_air_height(size_t n_hashes) {
    size_t h = 1;
    while (h < n_hashes * KA_ROUNDS) h <<= 1;
    return h;
}

template <int F> static int32_t ka_generate(p3gpu_ctx *ctx, const u64 *d_inputs, size_t n, u32 *d_trace) {
    const size_t height = keccak_air_height(n), blocks = (height + KA_ROUNDS - 1) / KA_ROUNDS;
    const unsigned threads = 32 * KA_GEN_WARPS;
    u32 *zero = nullptr;
    if (blocks > n) {                                               // padding rows: the zero-input block, computed once
        void *z = nullptr;
        P3_TRY(ctx_scratch2(ctx, (size_t)KA_ROUNDS * KA_COLS * 4, &z));
        zero = static_cast<u32 *>(z);
        keccak_air_generate_kernel<F><<<1, threads, 0, ctx->stream>>>(nullptr, 1, KA_ROUNDS, zero, nullptr);
        ctx->launches++;
    }
    keccak_air_generate_kernel<F><<<(unsigned)((blocks + KA_GEN_WARPS - 1) / KA_GEN_WARPS), threads, 0, ctx->stream>>>(d_inputs, n, height,
                                                                                                                       d_trace, zero);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t keccak_air_generate(p3gpu_ctx *ctx, int field, const u64 *d_inputs, size_t n_hashes, u32 *d_trace) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "Keccak AIR: unsupported field %d", field);
    P3_CHECK(n_hashes < ((size_t)1 << 40), P3GPU_EINVAL, "Keccak AIR: %zu hashes", n_hashes);
    return field == BABY_BEAR ? ka_generate<BABY_BEAR>(ctx, d_inputs, n_hashes, d_trace) : ka_generate<KOALA_BEAR>(ctx, d_inputs, n_hashes, d_trace);
}

int32_t keccak_air_quotient(p3gpu_ctx *ctx, int field, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q) {
    return air_hand_quotient(ctx, field, "Keccak", (const void *)keccak_air_quotient_kernel<BABY_BEAR>, (const void *)keccak_air_quotient_kernel<KOALA_BEAR>,
                             KA_CONSTRAINTS, KQ_WARPS, KQ_SMEM, AIR_USES_NEXT | AIR_USES_SELECTORS, d_lde, log_lde, log_n, alpha, d_q);
}

}  // namespace p3
