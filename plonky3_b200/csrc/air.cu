// Poseidon2 AIR on the device (SURVEY.md section 8f ranks 2 and 3): trace generation and quotient evaluation for
// VectorizedPoseidon2Air<F, WIDTH 16, SBOX_DEGREE, SBOX_REGISTERS, 4 + rounds_p + 4 rounds, VECTOR_LEN permutations per row>
// — the AIR of `prove_prime_field_31 --objective poseidon-2-permutations` (examples/examples/prove_prime_field_31.rs), in its
// two instances:
//   KoalaBear (BASELINE config 5): x^3 S-box, no register, 20 partial rounds, 164 columns per permutation
//   BabyBear: x^7 S-box with one register (the committed x^3; the S-box output is x3^2 x), 13 partial rounds, 298 columns
//
//   trace generation   poseidon2-air/src/generation.rs:14-70,184-253: one permutation ->
//                      inputs[16] | 4 x {sbox[16 REG], post[16]} | rounds_p x {sbox[REG], post_sbox} | 4 x {sbox[16 REG], post[16]};
//                      a vectorised row is VECTOR_LEN of them (REG = p2_reg<F>(), columns.rs)
//   constraints        poseidon2-air/src/air.rs:173-296, all of degree 3, no selectors: per full round the 16 register checks
//                      x3 - x^3 (REG = 1), then one assert_eq per post; per partial round the register check, then post_sbox;
//                      vectorised poseidon2-air/src/vectorized.rs:297-311
//   quotient           uni-stark/src/prover.rs:462-827: fold the constraints with powers of alpha (the first asserted constraint
//                      gets the highest power, uni-stark/src/folder.rs), multiply by 1/Z_H (commit/src/domain.rs:321-361)
//
// Both kernels are integer bound like the leaf sponge (one Poseidon2 evaluation per permutation); the quotient kernel also streams
// the 11 GB trace LDE once.  Mapping of the quotient kernel: 8 lanes per LDE row (one per permutation of the row, each reading its
// 656 contiguous bytes), constraints folded with lazy 64-bit multiply-accumulates against an alpha-power table in shared memory,
// 3-step shuffle reduction across the row's lanes.
#include "common.h"
#include "air_program.cuh"
#include "hash_core.cuh"

namespace p3 {

struct AirConsts {
    u32 beg[64], end[64], part[32];
    int rounds_p;
};
static_assert(sizeof(AirConsts) <= 1024, "kernel parameter budget");

constexpr int AIR_W = 16;
// S-box registers per S-box: the instance is a compile-time property of the field
template <int F> __host__ __device__ constexpr int p2_reg() { return F == BABY_BEAR ? 1 : 0; }
// columns / constraints of one permutation: 16 inputs + 8 full rounds x 16 (REG + 1) + rounds_p (REG + 1) (columns.rs)
__host__ __device__ constexpr size_t p2_cols(int reg, int rp) { return 16 + (size_t)(8 * AIR_W + rp) * (reg + 1); }
__host__ __device__ constexpr int p2_constraints(int reg, int rp) { return (8 * AIR_W + rp) * (reg + 1); }

template <int F> __device__ __forceinline__ void air_internal_layer(u32 (&s)[AIR_W]) {
    u32 part = s[1];
#pragma unroll
    for (int i = 2; i < AIR_W; i++) part = fp_add<F>(part, s[i]);
    const u32 sum = fp_add<F>(part, s[0]);
    s[0] = fp_sub<F>(part, s[0]);                       // V_0 = -2: -2 s0 + sum
    DiagLoop<F, AIR_W, 1>::run(s, sum);
}

// ---- trace generation: one thread per permutation, rows written through a per-warp shared-memory transpose ------------------
// A thread produces its permutation's 164 columns 16 (or rounds_p) at a time.  Written straight from the thread, a warp's store
// instruction touches 32 different rows 16 bytes each — partial sectors, and ncu shows the kernel stuck on the store queue
// (lg_throttle).  Instead every group of n values per permutation goes through a [32][n + 1] tile per warp and is
// written back with consecutive lanes on consecutive words of a row: whole 64/80-byte row segments per instruction.
//
// WINDOW: only columns [col0, col1) of the vectorised trace (rows of vec_len permutations) are stored, as a dense
// (n_perms / vec_len) x (col1 - col0) matrix — the column block one rank of the sharded prover commits.  Every permutation is
// still evaluated (its later columns depend on all earlier rounds); only the stores are filtered.

// REG = 1 (BabyBear): a full round is written as its 16 registers, then its 16 posts; the partial rounds' (register, post_sbox)
// pairs go through the tile 16 rounds (32 words per permutation) at a time.
template <int F, bool WINDOW>
__global__ void __launch_bounds__(128) p2air_generate_kernel(const u32 *inputs, size_t n_perms, u32 *trace, const __grid_constant__ AirConsts k,
                                                             const GenWindow win) {
    constexpr int REG = p2_reg<F>();
    __shared__ u32 tiles[4][32 * 33];
    u32 *tile = tiles[threadIdx.x >> 5];
    const unsigned lane = threadIdx.x & 31u;
    const size_t p0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) - lane;       // first permutation of this warp
    if (p0 >= n_perms) return;
    const size_t p = p0 + lane;
    const bool live = p < n_perms;
    const size_t cols = REG ? p2_cols(REG, k.rounds_p) : 144 + (size_t)k.rounds_p;
    const unsigned n_warp = (unsigned)min((size_t)32, n_perms - p0);
    // write `n` values per permutation (held as tile[perm * (n + 1) + i]) to columns [off, off + n) of the warp's rows
    auto flush = [&](unsigned n, size_t off) {
        __syncwarp();
        for (unsigned idx = lane; idx < n_warp * n; idx += 32) {
            const unsigned perm = idx / n, i = idx - perm * n;
            if constexpr (WINDOW) {
                const size_t pp = p0 + perm, c = (pp % win.vec_len) * cols + off + i;
                if (c >= win.col0 && c < win.col1) trace[(pp / win.vec_len) * (win.col1 - win.col0) + (c - win.col0)] = tile[perm * (n + 1) + i];
            } else {
                trace[(p0 + perm) * cols + off + i] = tile[perm * (n + 1) + i];
            }
        }
        __syncwarp();
    };
    u32 s[AIR_W];
    if (live) {
        const uint4 *ip = reinterpret_cast<const uint4 *>(inputs + p * 16);
#pragma unroll
        for (int i = 0; i < 4; i++) { const uint4 v = __ldg(ip + i); s[4 * i] = v.x; s[4 * i + 1] = v.y; s[4 * i + 2] = v.z; s[4 * i + 3] = v.w; }
    } else {
#pragma unroll
        for (int i = 0; i < AIR_W; i++) s[i] = 0;
    }
    auto put16 = [&](size_t off) {
#pragma unroll
        for (int i = 0; i < AIR_W; i++) tile[lane * 17 + i] = s[i];
        flush(16, off);
    };
    size_t off = 0;
    put16(off); off += 16;
    mds_light<F, AIR_W>(s);
    if constexpr (REG) {
        // x^7 through the committed register x3 = x^3: the S-box output is x3^2 x
        auto full = [&](const u32 *rc) {
#pragma unroll
            for (int i = 0; i < AIR_W; i++) {
                const u32 x = fp_add<F>(s[i], rc[i]), x3 = mont_mul<F>(mont_mul<F>(x, x), x);
                tile[lane * 17 + i] = x3;
                s[i] = mont_mul<F>(mont_mul<F>(x3, x3), x);
            }
            flush(16, off); off += 16;
            mds_light<F, AIR_W>(s);
            put16(off); off += 16;
        };
#pragma unroll 1
        for (int r = 0; r < 4; r++) full(k.beg + r * 16);
        const unsigned rp = (unsigned)k.rounds_p;
#pragma unroll 1
        for (unsigned r0 = 0; r0 < rp; r0 += 16) {
            const unsigned n = 2 * min(16u, rp - r0);
#pragma unroll 1
            for (unsigned r = r0; r < r0 + n / 2; r++) {
                const u32 x = fp_add<F>(s[0], k.part[r]), x3 = mont_mul<F>(mont_mul<F>(x, x), x);
                s[0] = mont_mul<F>(mont_mul<F>(x3, x3), x);
                tile[lane * (n + 1) + 2 * (r - r0)] = x3;
                tile[lane * (n + 1) + 2 * (r - r0) + 1] = s[0];
                air_internal_layer<F>(s);
            }
            flush(n, off); off += n;
        }
#pragma unroll 1
        for (int r = 0; r < 4; r++) full(k.end + r * 16);
    } else {
#pragma unroll 1
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int i = 0; i < AIR_W; i++) s[i] = sbox<F>(fp_add<F>(s[i], k.beg[r * 16 + i]));
            mds_light<F, AIR_W>(s);
            put16(off); off += 16;
        }
        const unsigned rp = (unsigned)k.rounds_p;
#pragma unroll 1
        for (unsigned r = 0; r < rp; r++) {
            s[0] = sbox<F>(fp_add<F>(s[0], k.part[r]));
            tile[lane * (rp + 1) + r] = s[0];
            air_internal_layer<F>(s);
        }
        flush(rp, off); off += rp;
#pragma unroll 1
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int i = 0; i < AIR_W; i++) s[i] = sbox<F>(fp_add<F>(s[i], k.end[r * 16 + i]));
            mds_light<F, AIR_W>(s);
            put16(off); off += 16;
        }
    }
}

// ---- quotient ----------------------------------------------------------------------------------------------------------
// One column segment of a sharded row block: columns [c0, c1) of the trace are a (rows x (c1 - c0)) row-major matrix at element
// offset `off` of the block.  c0 and c1 are multiples of 4, so a 16-byte load never straddles two segments.
struct QSeg { u32 c0, c1; u64 off; };
static_assert(sizeof(QSeg) == 16, "QSeg is one 16-byte shared-memory entry");
constexpr int QSEG_MAX = 512;

struct QuotArgs {
    const u32 *lde;      // H x (vec_len * cols), bit-reversed rows (SHARDED: this rank's row block, laid out by `segs`)
    u32 *q;              // H x 4, natural order over the quotient domain (SHARDED: rows x 4, the block's bit-reversed slice)
    const u32 *apow;     // (vec_len * n_constraints) EF4: alpha^j
    const u32 *invz;     // 2^rate_bits inverse vanishing values
    unsigned log_h, rate_mask;
    int vec_len;
    // SHARDED only
    const QSeg *segs;    // n_segs segments in column order, tiling [0, vec_len * cols)
    int n_segs;
    size_t row0, rows;   // the block is memory rows [row0, row0 + rows) of the bit-reversed LDE
};

// The BabyBear instance (REG = 1): one permutation's constraints folded into acc, c its first column, apv its alpha-power row.
// A permutation is 298 words = 1192 bytes, so every permutation starts 8-byte aligned: 8-byte loads throughout, and a partial
// round's (register, post_sbox) pair is one load.  Each register check is folded before the post check that follows it, in the
// constraint order of air.rs.
template <int F>
__device__ __forceinline__ void p2_fold_reg(const u32 *c, const uint4 *apv, const AirConsts &k, u64 (&acc)[4]) {
    const uint2 *c2 = reinterpret_cast<const uint2 *>(c);
    auto ld16 = [&](u32 (&dst)[AIR_W]) {
#pragma unroll
        for (int x = 0; x < 8; x++) { const uint2 w = __ldg(c2 + x); dst[2 * x] = w.x; dst[2 * x + 1] = w.y; }
        c2 += 8;
    };
    auto cube = [](u32 x) { return mont_mul<F>(mont_mul<F>(x, x), x); };
    u32 s[AIR_W];
    ld16(s);
    mds_light<F, AIR_W>(s);
    auto full = [&](const u32 *rc) {
        u32 w[AIR_W];
        ld16(w);                                                    // the 16 registers
#pragma unroll
        for (int x = 0; x < AIR_W; x++) {
            const u32 t = fp_add<F>(s[x], rc[x]);
            air_qmac<F>(acc, fp_sub<F>(w[x], cube(t)), apv[x]);
            s[x] = mont_mul<F>(mont_mul<F>(w[x], w[x]), t);
        }
        mds_light<F, AIR_W>(s);
        ld16(w);                                                    // the 16 posts
#pragma unroll
        for (int x = 0; x < AIR_W; x++) { air_qmac<F>(acc, fp_sub<F>(s[x], w[x]), apv[AIR_W + x]); s[x] = w[x]; }
        apv += 2 * AIR_W;
    };
#pragma unroll 1
    for (int r = 0; r < 4; r++) full(k.beg + r * 16);
#pragma unroll 1
    for (int r = 0; r < k.rounds_p; r++) {
        const uint2 w = __ldg(c2++);                                // (register, post_sbox)
        const u32 t = fp_add<F>(s[0], k.part[r]);
        air_qmac<F>(acc, fp_sub<F>(w.x, cube(t)), apv[0]);
        air_qmac<F>(acc, fp_sub<F>(mont_mul<F>(mont_mul<F>(w.x, w.x), t), w.y), apv[1]);
        apv += 2;
        s[0] = w.y;
        air_internal_layer<F>(s);
    }
#pragma unroll 1
    for (int r = 0; r < 4; r++) full(k.end + r * 16);
}

// SHARDED = false: the whole LDE, one thread per (natural index i, permutation v), reads memory row bitrev(i), writes q[i].
// SHARDED = true: one rank's row block of the row-sharded commit, one thread per (block row m, permutation v); memory row
// row0 + m is natural index i = bitrev(row0 + m), so it takes 1/Z_H entry i & rate_mask and writes q[m].  The block is read in
// place through the segment table (the chunk-major layout p3gpu_commit_sharded_dev leaves), never copied into a dense matrix.
// The BabyBear instance is dense only (p2_fold_reg per permutation).
// Threads per block: 128 for KoalaBear.  BabyBear's alpha table is 36 KB at vector_len 8; at 128 threads six blocks fill the SM's
// shared memory and leave L1 almost nothing, while every lane's 8-byte loads walk its own 1192-byte permutation and need L1 to keep
// the rest of each 32-byte sector.  512 threads share one table across 16 rows instead of 4.
template <int F> constexpr int p2q_block() { return p2_reg<F>() ? 512 : 128; }

template <int F, bool SHARDED>
__global__ void __launch_bounds__(p2q_block<F>()) p2air_quotient_kernel(const QuotArgs a, const __grid_constant__ AirConsts k) {
    constexpr int REG = p2_reg<F>();
    static_assert(!(REG && SHARDED), "the sharded quotient reads 16-byte units: KoalaBear only");
    // alpha powers, one padded row per permutation of the vector: constraint kk of permutation v (global index j = v * nc + kk,
    // multiplied by alpha^(n_all - 1 - j)) sits at ap[v * (nc + 1) + kk].  A quarter warp's 8 lanes are the 8 permutations of one
    // row, reading the same kk; 16-byte entries at a row stride of nc + 1 put lane v on banks 4 (v (nc + 1) mod 8) + 0..3, disjoint
    // for the 8 lanes exactly when nc + 1 is odd.  KoalaBear: nc + 1 = 149 (596 words = 20 mod 32); without the pad they collide 4
    // ways (ncu).  BabyBear: nc + 1 = 283 (1132 words = 12 mod 32), odd as well, so the same formula holds.
    extern __shared__ uint4 ap[];
    const int nc = REG ? p2_constraints(REG, k.rounds_p) : 128 + k.rounds_p, n_all = nc * a.vec_len;
    for (int t = threadIdx.x; t < n_all; t += blockDim.x) {
        const int j = n_all - 1 - t;
        ap[(j / nc) * (nc + 1) + (j % nc)] = __ldg(reinterpret_cast<const uint4 *>(a.apow) + t);
    }
    QSeg *sg = reinterpret_cast<QSeg *>(ap + a.vec_len * (nc + 1));   // SHARDED: the segment table behind the alpha powers
    if constexpr (SHARDED)
        for (int t = threadIdx.x; t < a.n_segs; t += blockDim.x) sg[t] = a.segs[t];
    __syncthreads();
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int lanes = a.vec_len;                                    // power of two <= 32 (checked by the host)
    const size_t i = t / lanes;                                     // SHARDED: the block row m
    const int v = (int)(t % lanes);
    const bool live = SHARDED ? i < a.rows : i < ((size_t)1 << a.log_h);
    u64 acc[4] = {0, 0, 0, 0};
    if constexpr (REG) {
        if (live) {
            const size_t m = (size_t)(__brevll((unsigned long long)i) >> (64 - a.log_h));
            p2_fold_reg<F>(a.lde + (m * lanes + v) * p2_cols(REG, k.rounds_p), ap + v * (nc + 1), k, acc);
        }
    } else if (live) {
        const size_t cols = 144 + (size_t)k.rounds_p;
        const size_t m = SHARDED ? i : (size_t)(__brevll((unsigned long long)i) >> (64 - a.log_h));
        const u32 *c = a.lde + (m * lanes + v) * cols;
        const uint4 *apv = ap + v * (nc + 1);
        // a permutation's 164 columns start 16-byte aligned (656 = 41 x 16 bytes): 16-byte loads throughout
        const uint4 *c4 = reinterpret_cast<const uint4 *>(c);
        // SHARDED: the permutation's columns are read in order; `c4` walks the current segment, `rem` columns are left in it
        int si = 0;
        u32 rem = 0;
        if constexpr (SHARDED) {
            const u32 col = (u32)(v * cols);
            int hi = a.n_segs - 1;
            while (si < hi) { const int mid = (si + hi) >> 1; if (sg[mid].c1 <= col) si = mid + 1; else hi = mid; }
            const QSeg s0 = sg[si];
            c4 = reinterpret_cast<const uint4 *>(a.lde + s0.off + m * (s0.c1 - s0.c0) + (col - s0.c0));
            rem = s0.c1 - col;
        }
        auto ldc = [&]() -> uint4 {                                 // SHARDED: next 4 columns of this permutation
            if (rem == 0) {
                const QSeg s1 = sg[++si];
                c4 = reinterpret_cast<const uint4 *>(a.lde + s1.off + m * (s1.c1 - s1.c0));
                rem = s1.c1 - s1.c0;
            }
            rem -= 4;
            return __ldg(c4++);
        };
        u32 s[AIR_W];
        auto ld16 = [&](u32 (&dst)[AIR_W]) {
            if constexpr (SHARDED) {
#pragma unroll
                for (int x = 0; x < 4; x++) { const uint4 v4 = ldc(); dst[4 * x] = v4.x; dst[4 * x + 1] = v4.y; dst[4 * x + 2] = v4.z; dst[4 * x + 3] = v4.w; }
            } else {
#pragma unroll
                for (int x = 0; x < 4; x++) { const uint4 v4 = __ldg(c4 + x); dst[4 * x] = v4.x; dst[4 * x + 1] = v4.y; dst[4 * x + 2] = v4.z; dst[4 * x + 3] = v4.w; }
                c4 += 4;
            }
        };
        ld16(s);
        mds_light<F, AIR_W>(s);
#pragma unroll 1
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int x = 0; x < AIR_W; x++) s[x] = sbox<F>(fp_add<F>(s[x], k.beg[r * 16 + x]));
            mds_light<F, AIR_W>(s);
            u32 post[AIR_W];
            ld16(post);
#pragma unroll
            for (int x = 0; x < AIR_W; x++) { air_qmac<F>(acc, fp_sub<F>(s[x], post[x]), apv[x]); s[x] = post[x]; }
            apv += 16;
        }
        {
            const u32 *cp = reinterpret_cast<const u32 *>(c4);
#pragma unroll 1
            for (int r = 0; r < k.rounds_p; r += 4) {           // rounds_p % 4 == 0 is checked by the host (20 for KoalaBear width 16)
                uint4 v4;
                if constexpr (SHARDED) v4 = ldc();
                else v4 = __ldg(reinterpret_cast<const uint4 *>(cp + r));
                const u32 pv[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
                for (int t2 = 0; t2 < 4; t2++) {
                    const u32 x3 = sbox<F>(fp_add<F>(s[0], k.part[r + t2]));
                    air_qmac<F>(acc, fp_sub<F>(x3, pv[t2]), *apv++);
                    s[0] = pv[t2];
                    air_internal_layer<F>(s);
                }
            }
            if constexpr (!SHARDED) c4 = reinterpret_cast<const uint4 *>(cp + k.rounds_p);
        }
#pragma unroll 1
        for (int r = 0; r < 4; r++) {
#pragma unroll
            for (int x = 0; x < AIR_W; x++) s[x] = sbox<F>(fp_add<F>(s[x], k.end[r * 16 + x]));
            mds_light<F, AIR_W>(s);
            u32 post[AIR_W];
            ld16(post);
#pragma unroll
            for (int x = 0; x < AIR_W; x++) { air_qmac<F>(acc, fp_sub<F>(s[x], post[x]), apv[x]); s[x] = post[x]; }
            apv += 16;
        }
    }
    u32 r[4];
#pragma unroll
    for (int d = 0; d < 4; d++) r[d] = mont_redc<F>(acc[d]);
    for (int off = 1; off < lanes; off <<= 1)
#pragma unroll
        for (int d = 0; d < 4; d++) r[d] = fp_add<F>(r[d], __shfl_xor_sync(0xffffffffu, r[d], off));
    if (live && v == 0) {
        const size_t nat = SHARDED ? (size_t)(__brevll((unsigned long long)(a.row0 + i)) >> (64 - a.log_h)) : i;
        const u32 z = __ldg(a.invz + (nat & a.rate_mask));
        reinterpret_cast<uint4 *>(a.q)[i] = make_uint4(mont_mul<F>(r[0], z), mont_mul<F>(r[1], z), mont_mul<F>(r[2], z), mont_mul<F>(r[3], z));
    }
}

// alpha^j, j < n (sequential per block of 32 with a square-and-multiply start)
template <int F> __global__ void ef_powers_kernel(u32 *pw, size_t n, const Ef4<F> alpha) {
    const size_t blk = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t j0 = blk * 32;
    if (j0 >= n) return;
    Ef4<F> cur; cur.c[0] = Fp<F>::ONE; cur.c[1] = cur.c[2] = cur.c[3] = 0;
    Ef4<F> base = alpha;
    for (size_t e = j0; e; e >>= 1) { if (e & 1) cur = ef_mul<F>(cur, base); base = ef_mul<F>(base, base); }
    for (size_t j = j0; j < n && j < j0 + 32; j++) {
        reinterpret_cast<uint4 *>(pw)[j] = make_uint4(cur.c[0], cur.c[1], cur.c[2], cur.c[3]);
        cur = ef_mul<F>(cur, alpha);
    }
}

static int32_t air_consts(p3gpu_ctx *ctx, int field, const AirConsts **out) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "Poseidon2 AIR: unsupported field %d", field);
    P3_CHECK(ctx->air_field >= 0, P3GPU_ESTATE, "Poseidon2 AIR round constants not set (p3gpu_p2air_set_constants)");
    P3_CHECK(ctx->air_field == field, P3GPU_ESTATE, "Poseidon2 AIR round constants were set for field %d, not %d", ctx->air_field, field);
    *out = reinterpret_cast<const AirConsts *>(ctx->air_consts);
    return P3GPU_OK;
}

// The row-sharded entry points read the trace in 16-byte units of 4-column segments; a BabyBear permutation is 298 columns, so
// every odd one starts in the middle of a unit.
int32_t air_sharded_field(int field) {
    P3_CHECK(field != BABY_BEAR, P3GPU_EUNSUPPORTED,
             "Poseidon2 AIR (BabyBear): no sharded prove: its 298-column permutations do not start on the 4-column units the sharded "
             "kernels read");
    return P3GPU_OK;
}

size_t air_columns(int field, int rounds_p) {
    if (field != BABY_BEAR && field != KOALA_BEAR) return 0;
    return p2_cols(field == BABY_BEAR ? p2_reg<BABY_BEAR>() : p2_reg<KOALA_BEAR>(), rounds_p);
}

int32_t air_set_constants(p3gpu_ctx *ctx, int field, const u32 *beg, const u32 *part, int rounds_p, const u32 *end) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "Poseidon2 AIR: unsupported field %d", field);
    // KoalaBear's quotient reads partial rounds four at a time with 16-byte loads; BabyBear's reads (register, post_sbox) pairs
    if (field == KOALA_BEAR)
        P3_CHECK(rounds_p >= 4 && rounds_p <= 32 && rounds_p % 4 == 0, P3GPU_EINVAL, "rounds_p %d must be a multiple of 4 in 4..32", rounds_p);
    else
        P3_CHECK(rounds_p >= 1 && rounds_p <= 32, P3GPU_EINVAL, "Poseidon2 AIR (BabyBear): rounds_p %d outside 1..32", rounds_p);
    static_assert(sizeof(AirConsts) <= sizeof(ctx->air_consts), "context storage for the AIR constants");
    const u32 P = field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    AirConsts k;
    memset(&k, 0, sizeof k);
    for (int i = 0; i < 64; i++) {
        P3_CHECK(beg[i] < P && end[i] < P, P3GPU_EINVAL, "round constant not in canonical Montgomery range");
        k.beg[i] = beg[i]; k.end[i] = end[i];
    }
    for (int i = 0; i < rounds_p; i++) { P3_CHECK(part[i] < P, P3GPU_EINVAL, "round constant not in canonical Montgomery range"); k.part[i] = part[i]; }
    k.rounds_p = rounds_p;
    memcpy(ctx->air_consts, &k, sizeof k);
    ctx->air_field = field;
    return P3GPU_OK;
}

int32_t air_generate_trace(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_perms, u32 *d_trace) {
    const AirConsts *k;
    P3_TRY(air_consts(ctx, field, &k));
    if (n_perms == 0) return P3GPU_OK;
    const unsigned grid = (unsigned)((n_perms + 127) / 128);
    if (field == BABY_BEAR) p2air_generate_kernel<BABY_BEAR, false><<<grid, 128, 0, ctx->stream>>>(d_inputs, n_perms, d_trace, *k, GenWindow{});
    else p2air_generate_kernel<KOALA_BEAR, false><<<grid, 128, 0, ctx->stream>>>(d_inputs, n_perms, d_trace, *k, GenWindow{});
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t air_generate_trace_cols(p3gpu_ctx *ctx, int field, int vec_len, const u32 *d_inputs, size_t n_perms, size_t col0, size_t col1, u32 *d_out) {
    const AirConsts *k;
    P3_TRY(air_consts(ctx, field, &k));
    P3_CHECK(vec_len >= 1 && n_perms % (size_t)vec_len == 0, P3GPU_EINVAL, "%zu permutations do not fill rows of %d", n_perms, vec_len);
    const size_t width = (size_t)vec_len * (144 + (size_t)k->rounds_p);
    P3_CHECK(col0 <= col1 && col1 <= width, P3GPU_EINVAL, "column window [%zu, %zu) outside the trace width %zu", col0, col1, width);
    if (n_perms == 0 || col0 == col1) return P3GPU_OK;
    const GenWindow win{col0, col1, (unsigned)vec_len};
    p2air_generate_kernel<KOALA_BEAR, true><<<(unsigned)((n_perms + 127) / 128), 128, 0, ctx->stream>>>(d_inputs, n_perms, d_out, *k, win);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

// The column segments of a row block as p3gpu_commit_sharded_dev leaves it: dense (one segment) with one rank, chunk-major
// otherwise — for every source rank g and every chunk [b, b') of shard_chunk_bounds(its block width), columns
// [col_starts[g] + b, col_starts[g] + b') at element offset rows * (col_starts[g] + b).
int32_t shard_col_segments(unsigned world, const size_t *col_starts, size_t rows, std::vector<size_t> &segs) {
    P3_CHECK(world >= 1 && world <= 16, P3GPU_EINVAL, "bad world %u", world);
    P3_CHECK(col_starts[0] == 0, P3GPU_EINVAL, "column blocks must start at 0");
    for (unsigned g = 0; g < world; g++) P3_CHECK(col_starts[g] <= col_starts[g + 1], P3GPU_EINVAL, "column blocks must be ordered");
    segs.clear();
    auto add = [&](size_t c0, size_t c1, size_t off) -> int32_t {
        P3_CHECK(c0 % 4 == 0 && c1 % 4 == 0, P3GPU_EINVAL,
                 "column segment [%zu, %zu) does not start and end on a multiple of 4 columns: a 16-byte load would straddle two chunks", c0, c1);
        P3_CHECK(c1 < (1ull << 32), P3GPU_EINVAL, "trace too wide");
        segs.insert(segs.end(), {c0, c1, off});
        return P3GPU_OK;
    };
    if (world == 1) {
        if (col_starts[1] > 0) P3_TRY(add(0, col_starts[1], 0));
    } else {
        for (unsigned g = 0; g < world; g++) {
            const std::vector<size_t> cb = shard_chunk_bounds(col_starts[g + 1] - col_starts[g]);
            for (size_t c = 0; c + 1 < cb.size(); c++)
                if (cb[c + 1] > cb[c]) P3_TRY(add(col_starts[g] + cb[c], col_starts[g] + cb[c + 1], rows * (col_starts[g] + cb[c])));
        }
    }
    P3_CHECK(segs.size() / 3 <= (size_t)QSEG_MAX, P3GPU_EUNSUPPORTED, "%zu column segments (at most %d)", segs.size() / 3, QSEG_MAX);
    return P3GPU_OK;
}

// alpha powers + 1/Z_H tables into scratch2, then one quotient launch (the whole LDE, or one row block with its segment table)
// (F, SHARDED) = (BABY_BEAR, true) is refused before this: the C ABI calls air_sharded_field first.
template <int F, bool SHARDED>
static int32_t quotient_launch(p3gpu_ctx *ctx, int field, int vec_len, const u32 *d_lde, unsigned log_h, unsigned log_n, const u32 *alpha, u32 *d_q,
                               const std::vector<size_t> *segs, size_t row0, size_t rows) {
    constexpr int REG = p2_reg<F>();
    const AirConsts *k;
    P3_TRY(air_consts(ctx, field, &k));
    P3_CHECK(vec_len >= 1 && vec_len <= 32 && (vec_len & (vec_len - 1)) == 0, P3GPU_EINVAL, "vector length %d must be a power of two <= 32", vec_len);
    P3_CHECK(log_h >= log_n && log_h <= Fp<F>::TWO_ADICITY && log_h - log_n <= 8, P3GPU_EINVAL, "bad domain sizes 2^%u / 2^%u", log_h, log_n);
    if constexpr (REG)                                              // the kernel's 8-byte LDE loads, 16-byte quotient stores
        P3_CHECK(reinterpret_cast<uintptr_t>(d_lde) % 8 == 0 && reinterpret_cast<uintptr_t>(d_q) % 16 == 0, P3GPU_EINVAL,
                 "quotient: the LDE must be 8-byte aligned, the quotient 16-byte aligned");
    else
        P3_CHECK(reinterpret_cast<uintptr_t>(d_lde) % 16 == 0 && reinterpret_cast<uintptr_t>(d_q) % 16 == 0, P3GPU_EINVAL, "quotient: buffers must be 16-byte aligned");
    const int nc = p2_constraints(REG, k->rounds_p), n_all = nc * vec_len;
    const unsigned rate_bits = log_h - log_n;
    const size_t nz = (size_t)1 << rate_bits;
    const size_t n_segs = SHARDED ? segs->size() / 3 : 0;
    if constexpr (SHARDED) {
        const size_t width = (size_t)vec_len * (144 + (size_t)k->rounds_p);
        P3_CHECK(n_segs > 0 && (*segs)[1 + 3 * (n_segs - 1)] == width, P3GPU_EINVAL, "the column blocks do not cover the trace width %zu", width);
        P3_CHECK(rows > 0 && row0 + rows <= ((size_t)1 << log_h), P3GPU_EINVAL, "row block [%zu, %zu) outside the LDE height 2^%u", row0, row0 + rows, log_h);
    }
    void *tab = nullptr;
    P3_TRY(ctx_scratch2(ctx, SHARDED ? (size_t)n_all * 16 + 256 * 4 + n_segs * sizeof(QSeg) : (size_t)n_all * 16 + nz * 4, &tab));
    u32 *apow = (u32 *)tab, *invz = apow + (size_t)n_all * 4;
    QSeg *dsegs = reinterpret_cast<QSeg *>(invz + 256);         // SHARDED: behind the largest 1/Z_H table, 16-byte aligned
    Ef4<F> al; for (int d = 0; d < 4; d++) al.c[d] = alpha[d];
    ef_powers_kernel<F><<<(unsigned)(((n_all + 31) / 32 + 63) / 64), 64, 0, ctx->stream>>>(apow, (size_t)n_all, al);
    std::vector<u32> zh, izh;                                       // Z_H and 1 / Z_H on the coset GENERATOR * K, by i mod 2^rate_bits
    air_domain<F>(log_h, log_n, 0, zh, izh);
    P3_CUDA(cudaMemcpyAsync(invz, izh.data(), nz * 4, cudaMemcpyHostToDevice, ctx->stream));
    QuotArgs qa;
    qa.lde = d_lde; qa.q = d_q; qa.apow = apow; qa.invz = invz; qa.log_h = log_h; qa.rate_mask = (unsigned)(nz - 1); qa.vec_len = vec_len;
    qa.segs = nullptr; qa.n_segs = 0; qa.row0 = row0; qa.rows = rows;
    if constexpr (SHARDED) {
        std::vector<QSeg> hs(n_segs);
        for (size_t s = 0; s < n_segs; s++) hs[s] = QSeg{(u32)(*segs)[3 * s], (u32)(*segs)[3 * s + 1], (u64)(*segs)[3 * s + 2]};
        P3_CUDA(cudaMemcpyAsync(dsegs, hs.data(), n_segs * sizeof(QSeg), cudaMemcpyHostToDevice, ctx->stream));
        qa.segs = dsegs; qa.n_segs = (int)n_segs;
    }
    const size_t threads = (SHARDED ? rows : (size_t)1 << log_h) * vec_len;
    const size_t smem = (size_t)vec_len * (nc + 1) * 16 + n_segs * sizeof(QSeg);
    auto kern = p2air_quotient_kernel<F, SHARDED>;
    if (smem > 48 * 1024) P3_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    constexpr int block = p2q_block<F>();
    kern<<<(unsigned)((threads + block - 1) / block), block, smem, ctx->stream>>>(qa, *k);
    ctx->launches += 2;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t air_quotient(p3gpu_ctx *ctx, int field, int vec_len, const u32 *d_lde, unsigned log_h, unsigned log_n, const u32 *alpha, u32 *d_q) {
    if (field == BABY_BEAR) return quotient_launch<BABY_BEAR, false>(ctx, field, vec_len, d_lde, log_h, log_n, alpha, d_q, nullptr, 0, 0);
    return quotient_launch<KOALA_BEAR, false>(ctx, field, vec_len, d_lde, log_h, log_n, alpha, d_q, nullptr, 0, 0);
}

int32_t air_quotient_sharded(p3gpu_ctx *ctx, int field, int vec_len, unsigned world, unsigned rank, const u32 *d_block, const size_t *col_starts,
                             unsigned log_h, unsigned log_n, const u32 *alpha, u32 *d_q) {
    const size_t H = (size_t)1 << log_h, rows = H / world;
    P3_CHECK(world >= 1 && rank < world && rows * world == H, P3GPU_EINVAL, "LDE height 2^%u does not split over %u ranks", log_h, world);
    std::vector<size_t> segs;
    P3_TRY(shard_col_segments(world, col_starts, rows, segs));
    return quotient_launch<KOALA_BEAR, true>(ctx, field, vec_len, d_block, log_h, log_n, alpha, d_q, &segs, (size_t)rank * rows, rows);
}

}  // namespace p3
