// Poseidon2 / Keccak-f sponges, SHA-256 and the Merkle-tree builder for sm_90a.
//
// Replaces MerkleTree::new (merkle-tree/src/merkle_tree.rs:95-178: first_digest_layer :268-338, compress :490-538,
// compress_and_inject :348-460) with the hash constructions the reference's MerkleTreeMmcs is instantiated with:
//   Poseidon2 (poseidon2/src/lib.rs:131-147, external.rs:60-159,288-336, monty-31/src/poseidon2.rs:76-85),
//   PaddingFreeSponge (symmetric/src/sponge.rs:182-216), TruncatedPermutation (symmetric/src/compression.rs:34-49),
//   KeccakF + SerializingHasher u64 packing (keccak/src/lib.rs:70-76, field/src/integers.rs:494-509),
//   CompressionFunctionFromHasher (symmetric/src/compression.rs:60-70),
//   SerializingHasher<Sha256> and Sha256Compress (symmetric/src/serializing_hasher.rs, sha256/src/lib.rs).
//
// Mapping: one sponge per thread (state in registers, rounds as loops so that a kernel stays inside the instruction cache, round
// constants passed as a __grid_constant__ kernel parameter = constant-bank operands).  The permutations themselves live in
// hash_core.cuh (also compiled and tested on the host).  These kernels are integer-ALU bound, not HBM bound (SURVEY.md §8d): a row
// of w elements costs ceil(w/RATE) permutations of ~4.3-5.6k integer instructions each against w*4 bytes of traffic.
#include <algorithm>
#include <cstring>

#include "common.h"
#include "hash_core.cuh"

namespace p3 {

template <int F, int W>
__global__ void __launch_bounds__(128) poseidon2_permute_kernel(u32 *states, size_t n, const __grid_constant__ Poseidon2Consts k) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    u32 s[W];
#pragma unroll
    for (int i = 0; i < W; i++) s[i] = states[idx * W + i];
    poseidon2_permute<F, W>(s, k);
#pragma unroll
    for (int i = 0; i < W; i++) states[idx * W + i] = s[i];
}

// ---- leaf sponge ---------------------------------------------------------------------------------
// The matrices of one height class (any number: merkle_tree.rs:131-133,312-316 has no limit).  Up to MAX_INLINE_MATS travel
// inside the kernel parameters (constant-bank operands); larger batches (commit_quotient with many chunks, batch-STARK style
// commits, one piece per source rank in the row-sharded multi-GPU commit) pass the table through device memory.
constexpr int MAX_INLINE_MATS = 8;
struct LeafArgs {
    const u32 *ptr[MAX_INLINE_MATS];
    u32 width[MAX_INLINE_MATS];
    int n_mats;
    size_t height;
    u32 *out;  // height x 8
    const u32 *const *dev_ptr;   // n_mats > MAX_INLINE_MATS: device arrays of n_mats pointers / widths, else null
    const u32 *dev_width;
    __device__ __forceinline__ const u32 *mat(int m) const { return dev_ptr ? dev_ptr[m] : ptr[m]; }
    __device__ __forceinline__ u32 wid(int m) const { return dev_ptr ? dev_width[m] : width[m]; }
};

// streaming cursor over the concatenation of row r of every matrix (input order; merkle_tree.rs:312-316)
struct RowCursor {
    const LeafArgs &a; size_t row; int m; u32 col, w; const u32 *p;
    __device__ __forceinline__ RowCursor(const LeafArgs &a_, size_t r) : a(a_), row(r), m(0), col(0), w(0), p(nullptr) { settle(); }
    __device__ __forceinline__ void settle() {
        while (m < a.n_mats && col >= (w = a.wid(m))) { m++; col = 0; }
        if (m < a.n_mats) p = a.mat(m) + row * w;
    }
    __device__ __forceinline__ bool more() const { return m < a.n_mats; }
    __device__ __forceinline__ u32 next() { u32 v = __ldg(p + col); col++; if (col >= w) settle(); return v; }
};

template <int F, int W>
__global__ void __launch_bounds__(128) poseidon2_leaf_kernel(const __grid_constant__ LeafArgs a, const __grid_constant__ Poseidon2Consts k) {
    constexpr int RATE = W - 8;
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.height) return;
    u32 s[W];
#pragma unroll
    for (int i = 0; i < W; i++) s[i] = 0;
    // one absorb/permute loop (a single inlined copy of the permutation) for both the one-matrix fast path and the
    // multi-matrix stream (rows concatenated in input order, merkle_tree.rs:312-316)
    const bool single = (a.n_mats == 1);
    const u32 w0 = a.width[0];
    const u32 *row0 = a.ptr[0] + r * w0;
    RowCursor cur(a, r);
    u32 c0 = 0;
    while (single ? (c0 < w0) : cur.more()) {
        if (single) {
#pragma unroll
            for (int i = 0; i < RATE; i++) if (c0 + i < w0) s[i] = __ldg(row0 + c0 + i);
            c0 += RATE;
        } else {
#pragma unroll
            for (int i = 0; i < RATE; i++) if (cur.more()) s[i] = cur.next();
        }
        poseidon2_permute<F, W>(s, k);
    }
    uint4 *o = reinterpret_cast<uint4 *>(a.out + r * 8);
    o[0] = make_uint4(s[0], s[1], s[2], s[3]);
    o[1] = make_uint4(s[4], s[5], s[6], s[7]);
}

// out[i] = perm16(left || right)[..8].  right == nullptr-equivalents are handled by the caller through `rmode`:
//   rmode 0: children are in[2i], in[2i+1]  (compress, merkle_tree.rs:490-538)
//   rmode 1: left = io[i] (in place), right = (i < inj_h ? inj[i] : 0)   (second compress of compress_and_inject)
template <int F>
__global__ void __launch_bounds__(128) poseidon2_compress_kernel(const u32 *in, const u32 *inj, size_t inj_h, u32 *out, size_t n, int rmode,
                                                                 const __grid_constant__ Poseidon2Consts k) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    u32 s[16];
    const uint4 *l = reinterpret_cast<const uint4 *>(rmode == 0 ? in + 16 * i : out + 8 * i);
    uint4 a = l[0], b = l[1], c, d;
    if (rmode == 0) { c = l[2]; d = l[3]; }
    else if (i < inj_h) { const uint4 *rp = reinterpret_cast<const uint4 *>(inj + 8 * i); c = rp[0]; d = rp[1]; }
    else { c = make_uint4(0, 0, 0, 0); d = c; }
    s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w; s[4] = b.x; s[5] = b.y; s[6] = b.z; s[7] = b.w;
    s[8] = c.x; s[9] = c.y; s[10] = c.z; s[11] = c.w; s[12] = d.x; s[13] = d.y; s[14] = d.z; s[15] = d.w;
    poseidon2_permute<F, 16>(s, k);
    uint4 *o = reinterpret_cast<uint4 *>(out + 8 * i);
    o[0] = make_uint4(s[0], s[1], s[2], s[3]);
    o[1] = make_uint4(s[4], s[5], s[6], s[7]);
}

// =================================================================================================
// Keccak-f[1600]
// =================================================================================================
__global__ void __launch_bounds__(128) keccak_f_kernel(u64 *states, size_t n) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n) return;
    KState s;
#pragma unroll
    for (int i = 0; i < 25; i++) { const u64 v = states[idx * 25 + i]; s.lo[i] = (u32)v; s.hi[i] = (u32)(v >> 32); }
    keccak_f(s);
#pragma unroll
    for (int i = 0; i < 25; i++) states[idx * 25 + i] = (u64)s.lo[i] | ((u64)s.hi[i] << 32);
}

// leaf = SerializingHasher<PaddingFreeSponge<KeccakF,25,17,4>>: u32 pairs -> u64 words over the concatenated row stream
// (field/src/integers.rs:494-509), overwrite-absorb 17 words per permutation (sponge.rs:182-216).
__global__ void __launch_bounds__(128) keccak_leaf_kernel(const __grid_constant__ LeafArgs a) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.height) return;
    KState s;
#pragma unroll
    for (int i = 0; i < 25; i++) { s.lo[i] = 0; s.hi[i] = 0; }
    const bool single = (a.n_mats == 1);
    const u32 w0 = a.width[0];
    const u32 *row0 = a.ptr[0] + r * w0;
    RowCursor cur(a, r);
    u32 c0 = 0;
    while (single ? (c0 < w0) : cur.more()) {
        if (single) {
#pragma unroll
            for (int i = 0; i < 17; i++) {
                const u32 e = c0 + 2 * i;
                if (e < w0) { s.lo[i] = __ldg(row0 + e); s.hi[i] = e + 1 < w0 ? __ldg(row0 + e + 1) : 0u; }
            }
            c0 += 34;
        } else {
#pragma unroll
            for (int i = 0; i < 17; i++) {
                if (cur.more()) {
                    s.lo[i] = cur.next();
                    s.hi[i] = cur.more() ? cur.next() : 0u;
                }
            }
        }
        keccak_f(s);
    }
    uint4 *o = reinterpret_cast<uint4 *>(a.out + r * 8);
    o[0] = make_uint4(s.lo[0], s.hi[0], s.lo[1], s.hi[1]);
    o[1] = make_uint4(s.lo[2], s.hi[2], s.lo[3], s.hi[3]);
}

// node = CompressionFunctionFromHasher<sponge,2,4>: 8 words < rate 17 -> exactly one permutation (compression.rs:60-70)
__global__ void __launch_bounds__(128) keccak_compress_kernel(const u32 *in, const u32 *inj, size_t inj_h, u32 *out, size_t n, int rmode) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    KState s;
#pragma unroll
    for (int j = 0; j < 25; j++) { s.lo[j] = 0; s.hi[j] = 0; }
    const uint4 *l = reinterpret_cast<const uint4 *>(rmode == 0 ? in + 16 * i : out + 8 * i);
    const uint4 a0 = l[0], a1 = l[1];
    s.lo[0] = a0.x; s.hi[0] = a0.y; s.lo[1] = a0.z; s.hi[1] = a0.w; s.lo[2] = a1.x; s.hi[2] = a1.y; s.lo[3] = a1.z; s.hi[3] = a1.w;
    uint4 b0 = make_uint4(0, 0, 0, 0), b1 = b0;
    if (rmode == 0) { b0 = l[2]; b1 = l[3]; }
    else if (i < inj_h) { const uint4 *rp = reinterpret_cast<const uint4 *>(inj + 8 * i); b0 = rp[0]; b1 = rp[1]; }
    s.lo[4] = b0.x; s.hi[4] = b0.y; s.lo[5] = b0.z; s.hi[5] = b0.w; s.lo[6] = b1.x; s.hi[6] = b1.y; s.lo[7] = b1.z; s.hi[7] = b1.w;
    keccak_f(s);
    uint4 *o = reinterpret_cast<uint4 *>(out + 8 * i);
    o[0] = make_uint4(s.lo[0], s.hi[0], s.lo[1], s.hi[1]);
    o[1] = make_uint4(s.lo[2], s.hi[2], s.lo[3], s.hi[3]);
}

// =================================================================================================
// SHA-256
// =================================================================================================
// leaf = SerializingHasher<Sha256> (symmetric/src/serializing_hasher.rs): the byte stream of the concatenated row is every element's
// to_unique_u32() — the Montgomery word — as 4 little-endian bytes (monty-31/src/monty_31.rs), so message word j is element j
// byte-swapped; 16 elements a block, then the padding of a message of `total` words.  One loop over the blocks, so the kernel holds
// one inlined copy of the compression.  The digest's bytes are the state words big-endian: word k = bswap(H[k]).
__global__ void __launch_bounds__(128) sha256_leaf_kernel(const __grid_constant__ LeafArgs a) {
    const size_t r = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= a.height) return;
    const bool single = (a.n_mats == 1);
    const u32 w0 = a.width[0];
    const u32 *row0 = a.ptr[0] + r * w0;
    u64 total = 0;
    for (int m = 0; m < a.n_mats; m++) total += a.wid(m);
    const u64 nb = sha256_blocks(total);
    RowCursor cur(a, r);
    u32 st[8];
    sha256_iv(st);
    for (u64 b = 0; b < nb; b++) {
        u32 w[16];
        const u64 j0 = 16 * b;
        if (single && j0 + 16 <= total) {                     // a whole block of one row: no per-word tests
#pragma unroll
            for (int i = 0; i < 16; i++) w[i] = bswap32(__ldg(row0 + j0 + i));
        } else {
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const u64 j = j0 + i;
                if (j < total) w[i] = bswap32(single ? __ldg(row0 + j) : cur.next());
                else w[i] = sha256_pad_word(j, total, nb, total * 32);
            }
        }
        sha256_compress(st, w);
    }
    uint4 *o = reinterpret_cast<uint4 *>(a.out + r * 8);
    o[0] = make_uint4(bswap32(st[0]), bswap32(st[1]), bswap32(st[2]), bswap32(st[3]));
    o[1] = make_uint4(bswap32(st[4]), bswap32(st[5]), bswap32(st[6]), bswap32(st[7]));
}

// node, same rmode convention as the other compress kernels.  The 64-byte block is left || right (each digest's bytes, i.e. its
// words byte-swapped).  HASHER: CompressionFunctionFromHasher<Sha256, 2, 32> (symmetric/src/compression.rs) = SHA-256 of the 64
// bytes: the block, then the constant padding block (0x80, zeros, bit length 512), whose message schedule folds to constants.
// Otherwise Sha256Compress (sha256/src/lib.rs): one compress256 of the block from H256_256, no padding.
template <bool HASHER>
__global__ void __launch_bounds__(128) sha256_compress_kernel(const u32 *in, const u32 *inj, size_t inj_h, u32 *out, size_t n, int rmode) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4 *l = reinterpret_cast<const uint4 *>(rmode == 0 ? in + 16 * i : out + 8 * i);
    const uint4 a0 = l[0], a1 = l[1];
    uint4 b0 = make_uint4(0, 0, 0, 0), b1 = b0;
    if (rmode == 0) { b0 = l[2]; b1 = l[3]; }
    else if (i < inj_h) { const uint4 *rp = reinterpret_cast<const uint4 *>(inj + 8 * i); b0 = rp[0]; b1 = rp[1]; }
    const u32 w[16] = {bswap32(a0.x), bswap32(a0.y), bswap32(a0.z), bswap32(a0.w), bswap32(a1.x), bswap32(a1.y), bswap32(a1.z), bswap32(a1.w),
                       bswap32(b0.x), bswap32(b0.y), bswap32(b0.z), bswap32(b0.w), bswap32(b1.x), bswap32(b1.y), bswap32(b1.z), bswap32(b1.w)};
    u32 st[8];
    sha256_iv(st);
    sha256_compress(st, w);
    if (HASHER) {
        const u32 pad[16] = {0x80000000u, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 512u};
        sha256_compress(st, pad);
    }
    uint4 *o = reinterpret_cast<uint4 *>(out + 8 * i);
    o[0] = make_uint4(bswap32(st[0]), bswap32(st[1]), bswap32(st[2]), bswap32(st[3]));
    o[1] = make_uint4(bswap32(st[4]), bswap32(st[5]), bswap32(st[6]), bswap32(st[7]));
}

// =================================================================================================
// host side
// =================================================================================================
static inline unsigned nblocks(size_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

static int32_t get_consts(p3gpu_ctx *ctx, int field, int width, const Poseidon2Consts **out) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    P3_CHECK(width == 16 || width == 24, P3GPU_EUNSUPPORTED, "Poseidon2 width %d unsupported (16 or 24)", width);
    const Poseidon2Consts *k = &ctx->p2_host[field][width == 24];
    P3_CHECK(k->set, P3GPU_ESTATE, "Poseidon2 constants for field %d width %d not set (p3gpu_poseidon2_set_constants)", field, width);
    *out = k;
    return P3GPU_OK;
}

int32_t hash_poseidon2_permute(p3gpu_ctx *ctx, int field, int width, u32 *d_states, size_t n) {
    const Poseidon2Consts *k;
    P3_TRY(get_consts(ctx, field, width, &k));
    if (n == 0) return P3GPU_OK;
    const unsigned g = nblocks(n, 128);
    if (field == BABY_BEAR && width == 16) poseidon2_permute_kernel<BABY_BEAR, 16><<<g, 128, 0, ctx->stream>>>(d_states, n, *k);
    else if (field == BABY_BEAR) poseidon2_permute_kernel<BABY_BEAR, 24><<<g, 128, 0, ctx->stream>>>(d_states, n, *k);
    else if (width == 16) poseidon2_permute_kernel<KOALA_BEAR, 16><<<g, 128, 0, ctx->stream>>>(d_states, n, *k);
    else poseidon2_permute_kernel<KOALA_BEAR, 24><<<g, 128, 0, ctx->stream>>>(d_states, n, *k);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t hash_keccak_f(p3gpu_ctx *ctx, u64 *d_states, size_t n) {
    if (n == 0) return P3GPU_OK;
    keccak_f_kernel<<<nblocks(n, 128), 128, 0, ctx->stream>>>(d_states, n);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

static int32_t launch_leaf(p3gpu_ctx *ctx, int field, int hash, const LeafArgs &a) {
    if (a.height == 0) return P3GPU_OK;
    const unsigned g = nblocks(a.height, 128);
    if (hash == P3GPU_HASH_KECCAK) {
        keccak_leaf_kernel<<<g, 128, 0, ctx->stream>>>(a);
    } else if (hash == P3GPU_HASH_SHA256 || hash == P3GPU_HASH_SHA256_COMPRESS) {
        sha256_leaf_kernel<<<g, 128, 0, ctx->stream>>>(a);
    } else {
        const Poseidon2Consts *k;
        P3_TRY(get_consts(ctx, field, hash == P3GPU_HASH_POSEIDON2_W24 ? 24 : 16, &k));
        if (field == BABY_BEAR && hash == P3GPU_HASH_POSEIDON2_W16) poseidon2_leaf_kernel<BABY_BEAR, 16><<<g, 128, 0, ctx->stream>>>(a, *k);
        else if (field == BABY_BEAR) poseidon2_leaf_kernel<BABY_BEAR, 24><<<g, 128, 0, ctx->stream>>>(a, *k);
        else if (hash == P3GPU_HASH_POSEIDON2_W16) poseidon2_leaf_kernel<KOALA_BEAR, 16><<<g, 128, 0, ctx->stream>>>(a, *k);
        else poseidon2_leaf_kernel<KOALA_BEAR, 24><<<g, 128, 0, ctx->stream>>>(a, *k);
    }
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

static int32_t launch_compress(p3gpu_ctx *ctx, int field, int hash, const u32 *in, const u32 *inj, size_t inj_h, u32 *out, size_t n, int rmode) {
    if (n == 0) return P3GPU_OK;
    const unsigned g = nblocks(n, 128);
    if (hash == P3GPU_HASH_KECCAK) {
        keccak_compress_kernel<<<g, 128, 0, ctx->stream>>>(in, inj, inj_h, out, n, rmode);
    } else if (hash == P3GPU_HASH_SHA256) {
        sha256_compress_kernel<true><<<g, 128, 0, ctx->stream>>>(in, inj, inj_h, out, n, rmode);
    } else if (hash == P3GPU_HASH_SHA256_COMPRESS) {
        sha256_compress_kernel<false><<<g, 128, 0, ctx->stream>>>(in, inj, inj_h, out, n, rmode);
    } else {
        const Poseidon2Consts *k;
        P3_TRY(get_consts(ctx, field, 16, &k));
        if (field == BABY_BEAR) poseidon2_compress_kernel<BABY_BEAR><<<g, 128, 0, ctx->stream>>>(in, inj, inj_h, out, n, rmode, *k);
        else poseidon2_compress_kernel<KOALA_BEAR><<<g, 128, 0, ctx->stream>>>(in, inj, inj_h, out, n, rmode, *k);
    }
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

static size_t next_pow2(size_t x) { size_t p = 1; while (p < x) p <<= 1; return p; }
static size_t padded_len2(size_t raw) { return raw <= 1 ? raw : (raw + 1) / 2 * 2; }  // merkle_tree.rs:473-481, N = 2

// mmcs/geometry.rs:83-124
static int32_t validate_heights(const size_t *hs, size_t n) {
    size_t maxh = 0;
    for (size_t i = 0; i < n; i++) maxh = std::max(maxh, hs[i]);
    P3_CHECK(maxh > 0, P3GPU_EINVAL, "all matrices have height 0");
    unsigned lmax = 0;
    while (((size_t)1 << lmax) < maxh) lmax++;
    for (size_t i = 0; i < n; i++) {
        unsigned l = 0;
        while (((size_t)1 << l) < hs[i]) l++;
        const size_t expect = hs[i] == 0 ? 1 : ((maxh - 1) >> (lmax - l)) + 1;
        P3_CHECK(hs[i] == expect, P3GPU_EINVAL, "matrix height %zu incompatible with tallest height %zu: expected %zu", hs[i], maxh, expect);
    }
    return P3GPU_OK;
}

int32_t hash_merkle_commit(p3gpu_ctx *ctx, int field, int hash, size_t n_mats, const u32 *const *d_mats, const size_t *heights,
                           const size_t *widths, u32 *d_layers, size_t *layer_lens, size_t *n_layers_out) {
    P3_CHECK(hash >= P3GPU_HASH_POSEIDON2_W16 && hash <= P3GPU_HASH_SHA256_COMPRESS, P3GPU_EUNSUPPORTED, "unknown hash %d", hash);
    P3_CHECK(n_mats >= 1, P3GPU_EINVAL, "No matrices given?");
    P3_TRY(validate_heights(heights, n_mats));
    for (size_t i = 0; i < n_mats; i++) P3_CHECK(widths[i] < (1ull << 31), P3GPU_EINVAL, "matrix width too large");
    // stable sort by height, tallest first (merkle_tree.rs:124-127)
    std::vector<size_t> order(n_mats);
    for (size_t i = 0; i < n_mats; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](size_t x, size_t y) { return heights[x] > heights[y]; });
    const size_t max_h = heights[order[0]];

    // device table for height classes with more than MAX_INLINE_MATS matrices: [n pointers][n widths] per class, every class
    // of this call in its own slice of one grow-only context buffer (classes of one call must not overwrite each other:
    // their kernels are only stream-ordered)
    size_t table_off = 0;
    void *table = nullptr;
    P3_TRY(ctx_leaf_table(ctx, n_mats * 16 + 64, &table));
    auto fill_leaf = [&](size_t begin, size_t end, size_t h, u32 *out, LeafArgs &la) -> int32_t {
        memset(&la, 0, sizeof la);
        std::vector<const u32 *> ps;
        std::vector<u32> ws;
        for (size_t k = begin; k < end; k++) {
            if (widths[order[k]] == 0) continue;  // contributes nothing to the stream
            ps.push_back(d_mats[order[k]]);
            ws.push_back((u32)widths[order[k]]);
        }
        la.n_mats = (int)ps.size();
        la.height = h; la.out = out;
        if (ps.size() <= (size_t)MAX_INLINE_MATS) {
            for (size_t k = 0; k < ps.size(); k++) { la.ptr[k] = ps[k]; la.width[k] = ws[k]; }
            return P3GPU_OK;
        }
        unsigned char *base = (unsigned char *)table + table_off;
        P3_CUDA(cudaMemcpyAsync(base, ps.data(), ps.size() * 8, cudaMemcpyHostToDevice, ctx->stream));           // pageable source: staged before return
        P3_CUDA(cudaMemcpyAsync(base + ps.size() * 8, ws.data(), ws.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
        la.dev_ptr = reinterpret_cast<const u32 *const *>(base);
        la.dev_width = reinterpret_cast<const u32 *>(base + ps.size() * 8);
        table_off += (ps.size() * 12 + 15) & ~(size_t)15;
        return P3GPU_OK;
    };

    size_t next = 0;
    while (next < n_mats && heights[order[next]] == max_h) next++;
    size_t n_layers = 0;
    u32 *cur = d_layers;
    size_t cur_len = padded_len2(max_h);
    if (cur_len > max_h) P3_CUDA(cudaMemsetAsync(cur + max_h * 8, 0, (cur_len - max_h) * 32, ctx->stream));
    {
        LeafArgs la;
        P3_TRY(fill_leaf(0, next, max_h, cur, la));
        P3_TRY(launch_leaf(ctx, field, hash, la));
    }
    layer_lens[n_layers++] = cur_len;
    while (cur_len > 1) {
        const size_t raw_next = cur_len / 2;
        const size_t next_layer_len = next_pow2(raw_next);
        const size_t inj_begin = next;
        while (next < n_mats && next_pow2(heights[order[next]]) == next_layer_len) next++;
        const size_t out_len = padded_len2(raw_next);
        u32 *out = cur + cur_len * 8;
        if (out_len > raw_next) P3_CUDA(cudaMemsetAsync(out + raw_next * 8, 0, (out_len - raw_next) * 32, ctx->stream));
        P3_TRY(launch_compress(ctx, field, hash, cur, nullptr, 0, out, raw_next, 0));
        if (next > inj_begin) {  // compress_and_inject (merkle_tree.rs:348-460)
            const size_t inj_h = heights[order[inj_begin]];
            void *rd = nullptr;
            P3_TRY(ctx_scratch2(ctx, inj_h * 32, &rd));
            LeafArgs la;
            P3_TRY(fill_leaf(inj_begin, next, inj_h, (u32 *)rd, la));
            P3_TRY(launch_leaf(ctx, field, hash, la));
            P3_TRY(launch_compress(ctx, field, hash, nullptr, (const u32 *)rd, inj_h, out, raw_next, 1));
        }
        P3_CHECK(n_layers < 64, P3GPU_EINVAL, "too many layers");
        layer_lens[n_layers++] = out_len;
        cur = out; cur_len = out_len;
    }
    *n_layers_out = n_layers;
    return P3GPU_OK;
}

// Layers above an existing digest layer (no matrices injected): used to finish a tree whose sub-tree roots were computed
// elsewhere (multi-GPU row sharding: every rank compresses the gathered sub-tree roots redundantly).
int32_t hash_merkle_from_digests(p3gpu_ctx *ctx, int field, int hash, const u32 *d_digests, size_t n, u32 *d_layers,
                                 size_t *layer_lens, size_t *n_layers_out) {
    P3_CHECK(hash >= P3GPU_HASH_POSEIDON2_W16 && hash <= P3GPU_HASH_SHA256_COMPRESS, P3GPU_EUNSUPPORTED, "unknown hash %d", hash);
    P3_CHECK(n >= 1, P3GPU_EINVAL, "no digests");
    size_t n_layers = 0;
    size_t cur_len = padded_len2(n);
    P3_CUDA(cudaMemcpyAsync(d_layers, d_digests, n * 32, cudaMemcpyDeviceToDevice, ctx->stream));
    if (cur_len > n) P3_CUDA(cudaMemsetAsync(d_layers + n * 8, 0, (cur_len - n) * 32, ctx->stream));
    u32 *cur = d_layers;
    layer_lens[n_layers++] = cur_len;
    while (cur_len > 1) {
        const size_t raw_next = cur_len / 2, out_len = padded_len2(raw_next);
        u32 *out = cur + cur_len * 8;
        if (out_len > raw_next) P3_CUDA(cudaMemsetAsync(out + raw_next * 8, 0, (out_len - raw_next) * 32, ctx->stream));
        P3_TRY(launch_compress(ctx, field, hash, cur, nullptr, 0, out, raw_next, 0));
        P3_CHECK(n_layers < 64, P3GPU_EINVAL, "too many layers");
        layer_lens[n_layers++] = out_len;
        cur = out; cur_len = out_len;
    }
    *n_layers_out = n_layers;
    return P3GPU_OK;
}

}  // namespace p3
