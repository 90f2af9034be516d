// Poseidon1 AIR on the device: trace generation and quotient evaluation for the reference's VectorizedPoseidon1Air<F, WIDTH 16,
// SBOX_DEGREE, SBOX_REGISTERS, 4, rounds_p, VECTOR_LEN> (poseidon1-air/src), the AIR of `prove_prime_field_31 -o
// poseidon-1-permutations` (examples/examples/prove_prime_field_31.rs), over BabyBear (x^7, one register: the committed x^3, the
// S-box output (x^3)^2 x) and KoalaBear (x^3, no register).  One template on the field serves both instances.
//
//   permutation        poseidon1/src/utils.rs optimized form: 4 full rounds (+ rc, S-box on all, circulant MDS), then
//                      + first_round_constants, the dense m_i once, rounds_p partial rounds (S-box on s0, + a scalar constant except
//                      in the last round, the sparse matrix {sparse_first_row[r], v[r]}), then 4 full rounds
//   trace generation   poseidon1-air/src/generation.rs: one permutation -> inputs[16] | 4 x {sbox regs[16 REG], post[16]} |
//                      rounds_p x {sbox regs[REG], post_sbox} | 4 x {regs, post}; a row holds vector_len permutations side by side
//   constraints        poseidon1-air/src/air.rs eval: per full round 16 register checks x3 - x^3 (REG = 1), then 16 checks
//                      mds_out - post; per partial round the register check, then sbox_out - post_sbox; degree 3, local row only
//   quotient           uni-stark/src/prover.rs:462-827 over GENERATOR * K, |K| = 2N, folded with alpha^(K - 1 - k), times 1 / Z_H
//
// Constants live in a device buffer of the context (p3gpu_p1air_set_constants): a header word rounds_p, then the P1_* sections
// below, compact (416 + 33 rounds_p words).  Every block stages them into shared memory once; both kernels are persistent.
#include "common.h"
#include "air_program.cuh"

namespace p3 {

constexpr int P1_W = 16, P1_RP_MAX = 32, P1_HDR = 4;
// sections (words after the header): initial full-round constants, terminal ones, the circulant MDS's first column (CANONICAL small
// integers), first_round_constants, m_i (row-major), sparse_first_row[rp][16], v[rp][16], the rp - 1 scalar round constants
constexpr int P1_INI = 0, P1_TER = 64, P1_CIRC = 128, P1_FRC = 144, P1_MI = 160, P1_SFR = 416;
constexpr u32 P1_CIRC_MAX = 1u << 12;   // circulant entries < 2^12: an MDS output row sums to < 16 * 2^12 * 2^31 = 2^47 < p 2^32
__host__ __device__ constexpr int p1_words(int rp) { return P1_SFR + 33 * rp; }
__host__ __device__ constexpr int p1_v(int rp) { return P1_SFR + 16 * rp; }
__host__ __device__ constexpr int p1_prc(int rp) { return P1_SFR + 32 * rp; }
template <int F> __host__ __device__ constexpr int p1_reg() { return F == BABY_BEAR ? 1 : 0; }
__host__ __device__ constexpr int p1_cols(int reg, int rp) { return P1_W + 8 * P1_W * (reg + 1) + rp * (reg + 1); }
__host__ __device__ constexpr int p1_constraints(int reg, int rp) { return 8 * P1_W * (reg + 1) + rp * (reg + 1); }

template <int F> __device__ __forceinline__ u32 p1_cube(u32 x) { return mont_mul<F>(mont_mul<F>(x, x), x); }

// acc += a b (Montgomery words), lazily: invariant acc < p 2^32, so mont_redc(acc) is the Montgomery form of the sum
template <int F> __device__ __forceinline__ void p1_mac(u64 &acc, u32 a, u32 b) {
    acc += (u64)a * b;
    u32 hi = (u32)(acc >> 32);
    const u32 hs = hi - Fp<F>::P;
    hi = hi < hs ? hi : hs;
    acc = ((u64)hi << 32) | (u32)acc;
}

// the full rounds' circulant MDS, s_i <- sum_j c[(i - j) mod 16] s_j with small canonical c: exact 64-bit sums, one reduction each
// (mont_redc(S) = S / R, times R^2 / R = S mod p: the sum keeps the Montgomery scaling of s)
template <int F> __device__ __forceinline__ void p1_circ_mds(u32 (&s)[P1_W], const u32 (&c)[P1_W]) {
    u32 o[P1_W];
#pragma unroll
    for (int i = 0; i < P1_W; i++) {
        u64 acc = 0;
#pragma unroll
        for (int j = 0; j < P1_W; j++) acc += (u64)c[(i - j) & 15] * s[j];
        o[i] = mont_mul<F>(mont_redc<F>(acc), Fp<F>::R2);
    }
#pragma unroll
    for (int i = 0; i < P1_W; i++) s[i] = o[i];
}

// s <- m s for the dense m_i (Montgomery, row-major in shared memory)
template <int F> __device__ __forceinline__ void p1_dense(u32 (&s)[P1_W], const u32 *m) {
    u32 o[P1_W];
#pragma unroll
    for (int i = 0; i < P1_W; i++) {
        u64 acc = 0;
#pragma unroll
        for (int j = 0; j < P1_W; j++) p1_mac<F>(acc, m[P1_W * i + j], s[j]);
        o[i] = mont_redc<F>(acc);
    }
#pragma unroll
    for (int i = 0; i < P1_W; i++) s[i] = o[i];
}

// the sparse matrix of partial round r with s0 the new state[0]: s0' = <first_row, (s0, s1..)>, s_i += s0 v[i - 1]
template <int F> __device__ __forceinline__ void p1_sparse(u32 (&s)[P1_W], u32 s0, const u32 *first_row, const u32 *v) {
    u64 acc = 0;
    p1_mac<F>(acc, first_row[0], s0);
#pragma unroll
    for (int j = 1; j < P1_W; j++) p1_mac<F>(acc, first_row[j], s[j]);
#pragma unroll
    for (int i = 1; i < P1_W; i++) s[i] = fp_add<F>(s[i], mont_mul<F>(s0, v[i - 1]));
    s[0] = mont_redc<F>(acc);
}

// ---- trace generation: one thread per permutation, rows written through a per-warp shared-memory transpose ----------------
// A warp's 32 permutations emit their columns in lockstep; each value goes to the warp's [32][33] tile, and every 32 columns the
// tile is written back with consecutive lanes on consecutive words of one permutation's columns: a 128-byte row segment per store
// instruction, instead of 32 rows 4 bytes each.
// WINDOW: only columns [win.col0, win.col1) of the vectorised trace (rows of win.vec_len permutations) are stored, as a dense
// (n_perms / vec_len) x (col1 - col0) matrix: the column block one rank of the sharded prover commits.  Every permutation is still
// evaluated; only the stores are filtered.
constexpr int P1G_WARPS = 8;

template <int F, bool WINDOW>
__global__ void __launch_bounds__(32 * P1G_WARPS, 2) p1air_generate_kernel(const u32 *inputs, size_t n_perms, u32 *trace, const u32 *kdev,
                                                                           const GenWindow win) {
    constexpr int REG = p1_reg<F>();
    extern __shared__ u32 p1g_sm[];
    const int rp = (int)__ldg(kdev);
    const int nk = p1_words(rp);
    for (int t = threadIdx.x; t < nk; t += blockDim.x) p1g_sm[t] = __ldg(kdev + P1_HDR + t);
    __syncthreads();
    const u32 *k = p1g_sm;
    const unsigned lane = threadIdx.x & 31u;
    u32 *tile = p1g_sm + ((nk + 3) & ~3) + (threadIdx.x >> 5) * (32 * 33);
    u32 c[P1_W];
#pragma unroll
    for (int i = 0; i < P1_W; i++) c[i] = k[P1_CIRC + i];
    const size_t cols = p1_cols(REG, rp);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t p0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x - lane; p0 < n_perms; p0 += stride) {
        const size_t p = p0 + lane;
        const bool live = p < n_perms;
        const unsigned n_warp = (unsigned)min((size_t)32, n_perms - p0);
        size_t off = 0;
        unsigned kk = 0;                                            // values in the tile (warp-uniform)
        auto flush = [&](unsigned n) {
            __syncwarp();
            for (unsigned idx = lane; idx < n_warp * n; idx += 32) {
                const unsigned perm = idx / n, i = idx - perm * n;
                if constexpr (WINDOW) {
                    const size_t pp = p0 + perm, c = (pp % win.vec_len) * cols + off + i;
                    if (c >= win.col0 && c < win.col1) trace[(pp / win.vec_len) * (win.col1 - win.col0) + (c - win.col0)] = tile[perm * 33 + i];
                } else {
                    trace[(p0 + perm) * cols + off + i] = tile[perm * 33 + i];
                }
            }
            __syncwarp();
            off += n;
            kk = 0;
        };
        auto put = [&](u32 v) {
            tile[lane * 33 + kk] = v;
            if (++kk == 32) flush(32);
        };
        u32 s[P1_W];
        if (live) {
            const uint4 *ip = reinterpret_cast<const uint4 *>(inputs + p * P1_W);
#pragma unroll
            for (int i = 0; i < 4; i++) { const uint4 v = __ldg(ip + i); s[4 * i] = v.x; s[4 * i + 1] = v.y; s[4 * i + 2] = v.z; s[4 * i + 3] = v.w; }
        } else {
#pragma unroll
            for (int i = 0; i < P1_W; i++) s[i] = 0;
        }
#pragma unroll
        for (int i = 0; i < P1_W; i++) put(s[i]);
        auto full = [&](const u32 *rc) {
#pragma unroll
            for (int i = 0; i < P1_W; i++) {
                const u32 t = fp_add<F>(s[i], rc[i]), x3 = p1_cube<F>(t);
                if constexpr (REG) { put(x3); s[i] = mont_mul<F>(mont_mul<F>(x3, x3), t); }
                else s[i] = x3;
            }
            p1_circ_mds<F>(s, c);
#pragma unroll
            for (int i = 0; i < P1_W; i++) put(s[i]);
        };
#pragma unroll 1
        for (int r = 0; r < 4; r++) full(k + P1_INI + P1_W * r);
#pragma unroll
        for (int i = 0; i < P1_W; i++) s[i] = fp_add<F>(s[i], k[P1_FRC + i]);
        p1_dense<F>(s, k + P1_MI);
#pragma unroll 1
        for (int r = 0; r < rp; r++) {
            const u32 t = s[0], x3 = p1_cube<F>(t);
            u32 o = x3;
            if constexpr (REG) { put(x3); o = mont_mul<F>(mont_mul<F>(x3, x3), t); }
            put(o);
            const u32 s0 = r < rp - 1 ? fp_add<F>(o, k[p1_prc(rp) + r]) : o;
            p1_sparse<F>(s, s0, k + P1_SFR + P1_W * r, k + p1_v(rp) + P1_W * r);
        }
#pragma unroll 1
        for (int r = 0; r < 4; r++) full(k + P1_TER + P1_W * r);
        if (kk) flush(kk);
    }
}

// ---- quotient --------------------------------------------------------------------------------------------------------------
// Persistent blocks of P1Q_WARPS warps; `lanes` (the vector length, a power of two <= 32) consecutive lanes share one point of the
// quotient domain, lane v evaluating permutation v of the row: it reads its own columns (KoalaBear: 164 words, 16-byte aligned,
// 16-byte loads; BabyBear: 298 words, so only every other permutation starts 16-byte aligned: 8-byte loads), runs the permutation
// on the committed values and folds its constraints with air_qmac against the alpha-power table in shared memory, laid out one
// padded row per permutation (stride nc + 1 entries: the 8 permutations of a quarter warp hit disjoint banks).  The row's lanes add
// their sums with a shuffle reduction; lane 0 multiplies by 1 / Z_H and stores q[i].
// SHARDED: one rank's chunk-major row block (AirHandQArgs); every load goes through the unit table behind the constants
// (air_program.cuh AirShardRow).  A 2- or 4-word load never leaves its 8-column unit, so a permutation that starts in the middle of
// a unit or a chunk (BabyBear: 298 columns) needs no split loads.
constexpr int P1Q_WARPS = 16;

template <int F, bool SHARDED> __global__ void __launch_bounds__(32 * P1Q_WARPS, 1) p1air_quotient_kernel(const AirHandQArgs a) {
    constexpr int REG = p1_reg<F>();
    constexpr int VEC = REG ? 2 : 4;                                    // words per load
    extern __shared__ uint4 p1q_sm[];
    const int rp = (int)__ldg(a.consts);
    const int nc = p1_constraints(REG, rp), cols = p1_cols(REG, rp);
    const int lanes = (int)a.lanes, n_all = nc * lanes;
    uint4 *ap = p1q_sm;
    u32 *k = reinterpret_cast<u32 *>(p1q_sm + lanes * (nc + 1));
    for (int t = threadIdx.x; t < n_all; t += blockDim.x) {
        const int v = t / nc;
        ap[v * (nc + 1) + (t - v * nc)] = __ldg(a.apow + t);
    }
    for (int t = threadIdx.x; t < p1_words(rp); t += blockDim.x) k[t] = __ldg(a.consts + P1_HDR + t);
    u64 *units = reinterpret_cast<u64 *>(k + ((p1_words(rp) + 1) & ~1));
    if constexpr (SHARDED) air_shard_table_load(a, units);
    __syncthreads();
    u32 c[P1_W];
#pragma unroll
    for (int i = 0; i < P1_W; i++) c[i] = k[P1_CIRC + i];
    const unsigned lane = threadIdx.x & 31u;
    const unsigned lshift = __ffs(lanes) - 1;
    const size_t total = SHARDED ? (size_t)a.rows << lshift : (size_t)1 << (a.d.log_q + lshift);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    // whole warps iterate together (the shuffles need every lane); lanes past the end only take part in them
    for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t - lane < total; t += stride) {
        const bool live = t < total;
        const u32 i = (u32)(t >> lshift);
        const int v = (int)(t & (lanes - 1));
        u64 acc[4] = {0, 0, 0, 0};
        if (live) {
            const u32 *row = SHARDED ? a.lde : a.lde + ((size_t)air_bitrev(i, a.d.log_q) * lanes + v) * cols;
            const AirShardRow sr{a.lde, units, i};
            const u32 pc = (u32)(v * cols);                         // SHARDED: the permutation's first column
            const uint4 *apv = ap + v * (nc + 1);
            auto fold = [&](u32 x) { air_qmac<F>(acc, x, *apv++); };
            auto ld1 = [&](int off) {
                if constexpr (SHARDED) return sr.ld(pc + off);
                else return __ldg(row + off);
            };
            auto ld16 = [&](u32 (&dst)[P1_W], int off) {
                if constexpr (SHARDED && VEC == 4) {
#pragma unroll
                    for (int x = 0; x < 4; x++) {
                        const uint4 w = __ldg(reinterpret_cast<const uint4 *>(sr.at(pc + off + 4 * x)));
                        dst[4 * x] = w.x; dst[4 * x + 1] = w.y; dst[4 * x + 2] = w.z; dst[4 * x + 3] = w.w;
                    }
                } else if constexpr (SHARDED) {
#pragma unroll
                    for (int x = 0; x < 8; x++) { const uint2 w = __ldg(reinterpret_cast<const uint2 *>(sr.at(pc + off + 2 * x))); dst[2 * x] = w.x; dst[2 * x + 1] = w.y; }
                } else if constexpr (VEC == 4) {
                    const uint4 *p4 = reinterpret_cast<const uint4 *>(row + off);
#pragma unroll
                    for (int x = 0; x < 4; x++) { const uint4 w = __ldg(p4 + x); dst[4 * x] = w.x; dst[4 * x + 1] = w.y; dst[4 * x + 2] = w.z; dst[4 * x + 3] = w.w; }
                } else {
                    const uint2 *p2 = reinterpret_cast<const uint2 *>(row + off);
#pragma unroll
                    for (int x = 0; x < 8; x++) { const uint2 w = __ldg(p2 + x); dst[2 * x] = w.x; dst[2 * x + 1] = w.y; }
                }
            };
            u32 s[P1_W];
            ld16(s, 0);
            auto full = [&](const u32 *rc, int off) {
                u32 sb[P1_W], w[P1_W];
                if constexpr (REG) ld16(w, off);
#pragma unroll
                for (int x = 0; x < P1_W; x++) {
                    const u32 tt = fp_add<F>(s[x], rc[x]), t3 = p1_cube<F>(tt);
                    if constexpr (REG) { fold(fp_sub<F>(w[x], t3)); sb[x] = mont_mul<F>(mont_mul<F>(w[x], w[x]), tt); }
                    else sb[x] = t3;
                }
                p1_circ_mds<F>(sb, c);
                ld16(w, off + P1_W * REG);
#pragma unroll
                for (int x = 0; x < P1_W; x++) { fold(fp_sub<F>(sb[x], w[x])); s[x] = w[x]; }
            };
            int off = P1_W;
#pragma unroll 1
            for (int r = 0; r < 4; r++, off += P1_W * (REG + 1)) full(k + P1_INI + P1_W * r, off);
#pragma unroll
            for (int x = 0; x < P1_W; x++) s[x] = fp_add<F>(s[x], k[P1_FRC + x]);
            p1_dense<F>(s, k + P1_MI);
#pragma unroll 1
            for (int r = 0; r < rp; r++, off += REG + 1) {
                const u32 tt = s[0], t3 = p1_cube<F>(tt);
                u32 o = t3;
                if constexpr (REG) {
                    const u32 x3 = ld1(off);
                    fold(fp_sub<F>(x3, t3));
                    o = mont_mul<F>(mont_mul<F>(x3, x3), tt);
                }
                const u32 post = ld1(off + REG);
                fold(fp_sub<F>(o, post));
                const u32 s0 = r < rp - 1 ? fp_add<F>(post, k[p1_prc(rp) + r]) : post;
                p1_sparse<F>(s, s0, k + P1_SFR + P1_W * r, k + p1_v(rp) + P1_W * r);
            }
#pragma unroll 1
            for (int r = 0; r < 4; r++, off += P1_W * (REG + 1)) full(k + P1_TER + P1_W * r, off);
        }
        u32 rr[4];
#pragma unroll
        for (int d = 0; d < 4; d++) rr[d] = mont_redc<F>(acc[d]);
        for (int o = 1; o < lanes; o <<= 1)
#pragma unroll
            for (int d = 0; d < 4; d++) rr[d] = fp_add<F>(rr[d], __shfl_xor_sync(0xffffffffu, rr[d], o));
        if (live && v == 0) {
            const u32 z = (SHARDED ? air_shard_odd(a, i) : i & 1u) ? a.izh[1] : a.izh[0];
#pragma unroll
            for (int d = 0; d < 4; d++) a.q[4 * (size_t)i + d] = mont_mul<F>(rr[d], z);
        }
    }
}

// ---- host entry points -------------------------------------------------------------------------------------------------------
static int p1_reg_of(int field) { return field == BABY_BEAR ? 1 : 0; }

size_t p1air_columns(int field, int rounds_p) {
    if (field != BABY_BEAR && field != KOALA_BEAR) return 0;
    return (size_t)p1_cols(p1_reg_of(field), rounds_p);
}

int32_t p1air_set_constants(p3gpu_ctx *ctx, int field, const u32 *ini, const u32 *ter, const u32 *circ, const u32 *frc, const u32 *mi, const u32 *prc,
                            const u32 *sfr, const u32 *v, int rp) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "Poseidon1 AIR: unsupported field %d", field);
    // KoalaBear's 16-byte column loads need every permutation and every full round 16-byte aligned: 144 + rounds_p = 0 mod 4
    if (field == KOALA_BEAR)
        P3_CHECK(rp >= 4 && rp <= P1_RP_MAX && rp % 4 == 0, P3GPU_EINVAL, "Poseidon1 AIR (KoalaBear): rounds_p %d must be a multiple of 4 in 4..%d", rp,
                 P1_RP_MAX);
    else
        P3_CHECK(rp >= 1 && rp <= P1_RP_MAX, P3GPU_EINVAL, "Poseidon1 AIR (BabyBear): rounds_p %d outside 1..%d", rp, P1_RP_MAX);
    const u32 P = field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    std::vector<u32> h(P1_HDR + p1_words(rp), 0);
    h[0] = (u32)rp;
    u32 *k = h.data() + P1_HDR;
    auto put = [&](int at, const u32 *src, int n, const char *what) -> int32_t {
        for (int i = 0; i < n; i++) {
            P3_CHECK(src[i] < P, P3GPU_EINVAL, "Poseidon1 AIR: %s[%d] is not a canonical Montgomery word", what, i);
            k[at + i] = src[i];
        }
        return P3GPU_OK;
    };
    P3_TRY(put(P1_INI, ini, 64, "initial_full"));
    P3_TRY(put(P1_TER, ter, 64, "terminal_full"));
    P3_TRY(put(P1_CIRC, circ, 16, "mds_circ_col"));
    P3_TRY(put(P1_FRC, frc, 16, "first_round_constants"));
    P3_TRY(put(P1_MI, mi, 256, "m_i"));
    P3_TRY(put(P1_SFR, sfr, 16 * rp, "sparse_first_row"));
    P3_TRY(put(p1_v(rp), v, 16 * rp, "v"));
    P3_TRY(put(p1_prc(rp), prc, rp - 1, "partial_rc"));
    for (int i = 0; i < 16; i++) {                                  // the kernels multiply by the canonical circulant entries
        const u32 cv = field == BABY_BEAR ? from_monty<BABY_BEAR>(circ[i]) : from_monty<KOALA_BEAR>(circ[i]);
        P3_CHECK(cv < P1_CIRC_MAX, P3GPU_EINVAL, "Poseidon1 AIR: mds_circ_col[%d] = %u: the kernels need circulant entries below %u", i, cv,
                 P1_CIRC_MAX);
        k[P1_CIRC + i] = cv;
    }
    if (!ctx->p1_consts) P3_CUDA(cudaMalloc(&ctx->p1_consts, (size_t)(P1_HDR + p1_words(P1_RP_MAX)) * 4));
    // on the context's stream: kernels queued before see the old constants, kernels queued after the new ones
    P3_CUDA(cudaMemcpyAsync(ctx->p1_consts, h.data(), h.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    ctx->p1_field = field;
    ctx->p1_rounds_p = rp;
    return P3GPU_OK;
}

static int32_t p1_state(p3gpu_ctx *ctx, int field) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "Poseidon1 AIR: unsupported field %d", field);
    P3_CHECK(ctx->p1_field >= 0, P3GPU_ESTATE, "Poseidon1 AIR constants not set (p3gpu_p1air_set_constants)");
    P3_CHECK(ctx->p1_field == field, P3GPU_ESTATE, "Poseidon1 AIR constants were set for field %d, not %d", ctx->p1_field, field);
    return P3GPU_OK;
}

template <int F, bool WINDOW> static int32_t p1_generate(p3gpu_ctx *ctx, const u32 *d_inputs, size_t n_perms, u32 *d_trace, const GenWindow &win) {
    const int nk = p1_words(ctx->p1_rounds_p);
    const size_t smem = (size_t)((nk + 3) & ~3) * 4 + (size_t)P1G_WARPS * 32 * 33 * 4;
    auto kern = p1air_generate_kernel<F, WINDOW>;
    P3_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    P3_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 32 * P1G_WARPS, smem));
    const size_t blocks = (n_perms + 32 * P1G_WARPS - 1) / (32 * P1G_WARPS);
    const unsigned grid = (unsigned)std::min<size_t>(blocks, (size_t)std::max(per_sm, 1) * ctx->sm_count);
    kern<<<grid, 32 * P1G_WARPS, smem, ctx->stream>>>(d_inputs, n_perms, d_trace, ctx->p1_consts, win);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t p1air_generate(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_perms, u32 *d_trace) {
    P3_TRY(p1_state(ctx, field));
    P3_CHECK(n_perms > 0, P3GPU_EINVAL, "Poseidon1 AIR: no permutations");
    P3_CHECK(reinterpret_cast<uintptr_t>(d_inputs) % 16 == 0 && reinterpret_cast<uintptr_t>(d_trace) % 4 == 0, P3GPU_EINVAL,
             "Poseidon1 AIR trace: inputs must be 16-byte aligned, the trace 4-byte aligned");
    const GenWindow win{};
    return field == BABY_BEAR ? p1_generate<BABY_BEAR, false>(ctx, d_inputs, n_perms, d_trace, win)
                              : p1_generate<KOALA_BEAR, false>(ctx, d_inputs, n_perms, d_trace, win);
}

int32_t p1air_generate_cols(p3gpu_ctx *ctx, int field, int vector_len, const u32 *d_inputs, size_t n_perms, size_t col0, size_t col1, u32 *d_out) {
    P3_TRY(p1_state(ctx, field));
    P3_CHECK(vector_len >= 1 && vector_len <= 32 && n_perms > 0 && n_perms % (size_t)vector_len == 0, P3GPU_EINVAL,
             "Poseidon1 AIR: %zu permutations do not fill rows of %d", n_perms, vector_len);
    P3_CHECK(reinterpret_cast<uintptr_t>(d_inputs) % 16 == 0 && reinterpret_cast<uintptr_t>(d_out) % 4 == 0, P3GPU_EINVAL,
             "Poseidon1 AIR trace: inputs must be 16-byte aligned, the trace 4-byte aligned");
    P3_TRY(air_check_window("Poseidon1", col0, col1, (size_t)vector_len * p1air_columns(field, ctx->p1_rounds_p)));
    if (col0 == col1) return P3GPU_OK;
    const GenWindow win{col0, col1, (unsigned)vector_len};
    return field == BABY_BEAR ? p1_generate<BABY_BEAR, true>(ctx, d_inputs, n_perms, d_out, win)
                              : p1_generate<KOALA_BEAR, true>(ctx, d_inputs, n_perms, d_out, win);
}

static int32_t p1_quotient(p3gpu_ctx *ctx, int field, int vector_len, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q,
                           const AirHandShard *shard) {
    P3_TRY(p1_state(ctx, field));
    P3_CHECK(vector_len >= 1 && vector_len <= 32 && (vector_len & (vector_len - 1)) == 0, P3GPU_EINVAL,
             "Poseidon1 AIR quotient: vector length %d must be a power of two <= 32", vector_len);
    const int reg = p1_reg_of(field), rp = ctx->p1_rounds_p;
    const unsigned lde_align = reg ? 8 : 16;                          // the kernel's load width
    P3_CHECK(reinterpret_cast<uintptr_t>(d_lde) % lde_align == 0, P3GPU_EINVAL, "Poseidon1 AIR quotient: the LDE must be %u-byte aligned", lde_align);
    const int nc = p1_constraints(reg, rp);
    if (!shard) {
        const size_t smem = (size_t)vector_len * (nc + 1) * 16 + (size_t)p1_words(rp) * 4;
        return air_hand_quotient(ctx, field, "Poseidon1", (const void *)p1air_quotient_kernel<BABY_BEAR, false>,
                                 (const void *)p1air_quotient_kernel<KOALA_BEAR, false>, (u32)(nc * vector_len), P1Q_WARPS, smem, 0, d_lde, log_lde,
                                 log_n, alpha, d_q, ctx->p1_consts, (unsigned)vector_len);
    }
    const size_t smem = (size_t)vector_len * (nc + 1) * 16 + (size_t)((p1_words(rp) + 1) & ~1) * 4;   // the unit table 8-byte aligned behind
    const AirHandShard sh{shard->world, shard->rank, shard->col_starts, (size_t)vector_len * p1_cols(reg, rp)};
    return air_hand_quotient(ctx, field, "Poseidon1", (const void *)p1air_quotient_kernel<BABY_BEAR, true>,
                             (const void *)p1air_quotient_kernel<KOALA_BEAR, true>, (u32)(nc * vector_len), P1Q_WARPS, smem, 0, d_lde, log_lde, log_n,
                             alpha, d_q, ctx->p1_consts, (unsigned)vector_len, &sh);
}

int32_t p1air_quotient(p3gpu_ctx *ctx, int field, int vector_len, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q) {
    return p1_quotient(ctx, field, vector_len, d_lde, log_lde, log_n, alpha, d_q, nullptr);
}

int32_t p1air_quotient_sharded(p3gpu_ctx *ctx, int field, int vector_len, const AirHandShard &shard, const u32 *d_block, unsigned log_lde,
                               unsigned log_n, const u32 *alpha, u32 *d_q) {
    return p1_quotient(ctx, field, vector_len, d_block, log_lde, log_n, alpha, d_q, &shard);
}

}  // namespace p3
