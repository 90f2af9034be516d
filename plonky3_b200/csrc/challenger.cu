// Device-resident Fiat-Shamir transcript: DuplexChallenger<F, Poseidon2, WIDTH, RATE> (challenger/src/duplex_challenger.rs:60-114,
// 168-300) and its proof-of-work grinding (challenger/src/grinding_challenger.rs:100-232).
//
// The reference keeps the transcript on the host.  With the prover's data resident on the GPU the values it has to absorb (Merkle
// caps, thousands of opened values) are produced on the device, so the sponge lives there too: its state, input and output
// buffers sit in device memory, `observe` is one single-thread kernel walking a device (or staged host) slice through the sponge —
// a few microseconds per permutation, no PCIe round trip per duplexing — and `sample` copies squeezed elements back.  Grinding is a
// parallel search over candidate witnesses (every thread permutes `transcript || candidate`, the smallest valid witness wins —
// what a serial reference build returns; parallel builds may return any valid one, SURVEY 8c "Determinism caveat").
// This is protocol plumbing for the config-5 prove driver (SURVEY 8f / N1), not part of the hot path.
#include "common.h"
#include "hash_core.cuh"

//
// The second kind of handle is SerializingChallenger32<F, HashChallenger<u8, Keccak256Hash, 32>> (challenger/src/
// serializing_challenger.rs, hash_challenger.rs), the transcript of the Keccak configuration (examples/src/types.rs:19-35).  The
// reference keeps every observed byte in an input buffer and hashes all of it when a sample finds the output buffer empty; the
// digest then becomes both the new input buffer and the output buffer, whose bytes are popped from the end.  Absorbing the input
// block by block as it fills gives the same digest, so the device keeps a running Keccak state plus the pending partial block (at
// most 33 words: every input is a whole number of 32-bit words) instead of a buffer that grows with the opened values.
//
// The third kind is the same HashChallenger over Sha256 (sha256/src/lib.rs), the transcript of the SHA-256 configurations
// (keccak-air/examples/prove_baby_bear_sha256*.rs): the SHA-256 midstate over the full 64-byte blocks, the pending big-endian message
// words of the partial block (at most 15), the number of full blocks (for the length in the padding) and the output buffer.
struct p3gpu_challenger {
    int kind;           // CH_DUPLEX, CH_KECCAK256 or CH_SHA256
    int field, width, rate;
    p3::u32 *state;     // device, duplex: [0, width) sponge state | [32, 32+rate) input buffer | [64, 64+rate) output buffer | [96] n_in | [97] n_out
                        //         keccak: [0, 50) Keccak state (lo[25], hi[25]) | [64, 98) pending words | [98] n_pending | [100, 108) output words | [108] n_out words
                        //         sha256: [0, 8) midstate | [8] full blocks | [64, 80) pending words | [98] n_pending | [100, 108) output = H[0..8) | [108] n_out words
    p3::u32 *stage;     // device staging for host observes / samples (4096 words)
};

namespace p3 {

constexpr int CH_DUPLEX = 0, CH_KECCAK256 = 1, CH_SHA256 = 2;
constexpr int CH_IN = 32, CH_OUT = 64, CH_NIN = 96, CH_NOUT = 97, CH_WORDS = 128, CH_STAGE = 4096;
constexpr int KCH_PEND = 64, KCH_NPEND = 98, KCH_OUT = 100, KCH_NOUT = 108, SCH_BLOCKS = 8;

template <int F, int W>
__device__ void ch_duplexing(u32 *st, int rate, const Poseidon2Consts &k) {
    const u32 n = st[CH_NIN];
    u32 s[W];
#pragma unroll
    for (int i = 0; i < W; i++) s[i] = st[i];
    if (n > 0) {
#pragma unroll
        for (int i = 0; i < W; i++)
            if (i < rate) s[i] = (u32)i < n ? st[CH_IN + i] : 0u;           // overwrite the leading rate slots, clear the rest of the rate
        s[rate] = fp_add<F>(s[rate], to_monty<F>(n));                       // bind the absorbed length into the first capacity element
    }
    poseidon2_permute<F, W>(s, k);
#pragma unroll
    for (int i = 0; i < W; i++) st[i] = s[i];
    for (int i = 0; i < rate; i++) st[CH_OUT + i] = s[i];
    st[CH_NIN] = 0; st[CH_NOUT] = (u32)rate;
}

template <int F, int W>
__global__ void ch_observe_kernel(u32 *st, int rate, const u32 *vals, size_t n, const __grid_constant__ Poseidon2Consts k) {
    if (threadIdx.x | blockIdx.x) return;
    for (size_t j = 0; j < n; j++) {
        st[CH_NOUT] = 0;                                                      // any buffered output is now invalid
        const u32 m = st[CH_NIN];
        st[CH_IN + m] = vals[j];
        st[CH_NIN] = m + 1;
        if (m + 1 == (u32)rate) ch_duplexing<F, W>(st, rate, k);
    }
}

template <int F, int W>
__global__ void ch_sample_kernel(u32 *st, int rate, u32 *out, size_t n, const __grid_constant__ Poseidon2Consts k) {
    if (threadIdx.x | blockIdx.x) return;
    for (size_t j = 0; j < n; j++) {
        if (st[CH_NIN] != 0 || st[CH_NOUT] == 0) ch_duplexing<F, W>(st, rate, k);
        const u32 m = st[CH_NOUT] - 1;                                        // samples pop from the END of the output buffer
        out[j] = st[CH_OUT + m];
        st[CH_NOUT] = m;
    }
}

// candidate c is valid iff the sample after observing it has `bits` trailing zero bits (canonical value); best = smallest valid c
template <int F, int W>
__global__ void __launch_bounds__(128) ch_grind_kernel(const u32 *st, int rate, u32 base, u32 count, u32 mask, u32 *best, const __grid_constant__ Poseidon2Consts k) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const u32 cand = base + t;
    if (cand >= Fp<F>::P) return;
    const u32 widx = st[CH_NIN];
    u32 s[W];
#pragma unroll
    for (int i = 0; i < W; i++) {
        if (i < rate) s[i] = (u32)i < widx ? st[CH_IN + i] : 0u;
        else s[i] = st[i];
    }
#pragma unroll
    for (int i = 0; i < W; i++) if ((u32)i == widx) s[i] = to_monty<F>(cand);
    s[rate] = fp_add<F>(s[rate], to_monty<F>(widx + 1));
    poseidon2_permute<F, W>(s, k);
    u32 last = 0;
#pragma unroll
    for (int i = 0; i < W; i++) if (i == rate - 1) last = s[i];
    if ((from_monty<F>(last) & mask) == 0) atomicMin(best, cand);
}

// ---- SerializingChallenger32<F, HashChallenger<u8, Keccak256Hash, 32>> ------------------------------------------------------
__device__ __forceinline__ void kch_load(const u32 *st, KState &s) {
#pragma unroll
    for (int i = 0; i < 25; i++) { s.lo[i] = st[i]; s.hi[i] = st[25 + i]; }
}
__device__ __forceinline__ void kch_store(u32 *st, const KState &s) {
#pragma unroll
    for (int i = 0; i < 25; i++) { st[i] = s.lo[i]; st[25 + i] = s.hi[i]; }
}
__device__ __forceinline__ void kch_full_block(u32 *st, KState &s) {
    u32 w[KECCAK256_RATE_WORDS];
#pragma unroll
    for (int i = 0; i < KECCAK256_RATE_WORDS; i++) w[i] = st[KCH_PEND + i];
    keccak256_absorb_block(s, w);
    st[KCH_NPEND] = 0;
}

// HashChallenger::flush: digest of everything observed; the digest is the new input buffer and the output buffer
__device__ void kch_flush(u32 *st) {
    KState s;
    kch_load(st, s);
    u32 w[KECCAK256_RATE_WORDS];
#pragma unroll
    for (int i = 0; i < KECCAK256_RATE_WORDS; i++) w[i] = st[KCH_PEND + i];
    keccak256_final_block(s, w, st[KCH_NPEND]);
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const u32 d = keccak256_digest_word(s, k);
        st[KCH_PEND + k] = d;
        st[KCH_OUT + k] = d;
    }
    for (int i = 0; i < 50; i++) st[i] = 0;
    st[KCH_NPEND] = 8;
    st[KCH_NOUT] = 8;
}

// four bytes popped from the END of the output buffer, as u32::from_le_bytes of the popped order (bytes 31, 30, 29, 28 first)
__device__ __forceinline__ u32 kch_pop_u32(u32 *st) {
    if (st[KCH_NOUT] == 0) kch_flush(st);
    const u32 m = st[KCH_NOUT] - 1;
    st[KCH_NOUT] = m;
    return __byte_perm(st[KCH_OUT + m], 0, 0x0123);
}

// MONTY: observe Montgomery words as the 4 little-endian bytes of their canonical values (CanObserve<F>); otherwise the words'
// own bytes (a [u64; 4] digest held as 8 words)
template <int F, bool MONTY>
__global__ void kch_observe_kernel(u32 *st, const u32 *vals, size_t n) {
    if (threadIdx.x | blockIdx.x) return;
    if (n == 0) return;
    KState s;
    kch_load(st, s);
    st[KCH_NOUT] = 0;                                                          // any buffered output is now invalid
    u32 m = st[KCH_NPEND];
    for (size_t j = 0; j < n; j++) {
        st[KCH_PEND + m] = MONTY ? from_monty<F>(vals[j]) : vals[j];
        if (++m == (u32)KECCAK256_RATE_WORDS) { kch_full_block(st, s); m = 0; }
    }
    st[KCH_NPEND] = m;
    kch_store(st, s);
}

// raw = false: field elements by rejection sampling of 31-bit values (CanSample<F>), returned as Montgomery words; raw = true: the
// u32 of 4 popped bytes AND `mask` (CanSampleBits)
template <int F>
__global__ void kch_sample_kernel(u32 *st, u32 *out, size_t n, bool raw, u32 mask) {
    if (threadIdx.x | blockIdx.x) return;
    for (size_t j = 0; j < n; j++) {
        if (raw) { out[j] = kch_pop_u32(st) & mask; continue; }
        u32 v;
        do { v = kch_pop_u32(st) & 0x7fffffffu; } while (v >= Fp<F>::P);
        out[j] = to_monty<F>(v);
    }
}

// Candidate c is valid iff observe(c); sample_bits(bits) == 0.  The full blocks of the transcript are already absorbed (the
// midstate); every thread absorbs the pending words, its candidate and the padding — one or two Keccak-f — and takes the first
// sampled u32, which is the byte-reversed last digest word.  best = smallest valid c.
template <int F>
__global__ void __launch_bounds__(128) kch_grind_kernel(const u32 *st, u32 base, u32 count, u32 mask, u32 *best) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const u32 cand = base + t;
    if (cand >= Fp<F>::P) return;
    const u32 n = st[KCH_NPEND];
    KState s;
    kch_load(st, s);
    u32 w[KECCAK256_RATE_WORDS];
#pragma unroll
    for (int i = 0; i < KECCAK256_RATE_WORDS; i++) w[i] = (u32)i < n ? st[KCH_PEND + i] : ((u32)i == n ? cand : 0u);
    u32 tail = n + 1;
    if (tail == (u32)KECCAK256_RATE_WORDS) { keccak256_absorb_block(s, w); tail = 0; }
    keccak256_final_block(s, w, tail);
    const u32 sample = __byte_perm(keccak256_digest_word(s, 7), 0, 0x0123);
    if ((sample & mask) == 0) atomicMin(best, cand);
}

// ---- SerializingChallenger32<F, HashChallenger<u8, Sha256, 32>> ------------------------------------------------------------
// The tail of the message after the full blocks: `n` pending words, then `extra` (if has_extra), then the padding for a message of
// `blocks` full blocks plus the tail.  One or two compressions from the midstate `h`; one inlined copy of the compression.
__device__ __forceinline__ void sch_finish(u32 (&h)[8], const u32 *pend, u32 n, bool has_extra, u32 extra, u32 blocks) {
    const u32 tail = n + (has_extra ? 1u : 0u);
    const u64 nb = sha256_blocks(tail), bits = ((u64)blocks * 16 + tail) * 32;
#pragma unroll 1
    for (u64 b = 0; b < nb; b++) {
        u32 w[16];
#pragma unroll
        for (int i = 0; i < 16; i++) {
            const u64 j = 16 * b + i;
            w[i] = j < n ? pend[i] : (j < tail ? extra : sha256_pad_word(j, tail, nb, bits));
        }
        sha256_compress(h, w);
    }
}

// HashChallenger::flush: the digest's bytes are H big-endian; they become the new input buffer (8 message words = H, the midstate
// back at the IV) and the output buffer
__device__ void sch_flush(u32 *st) {
    u32 h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = st[i];
    sch_finish(h, st + KCH_PEND, st[KCH_NPEND], false, 0, st[SCH_BLOCKS]);
#pragma unroll
    for (int k = 0; k < 8; k++) { st[KCH_PEND + k] = h[k]; st[KCH_OUT + k] = h[k]; st[k] = SHA256_IV[k]; }
    st[SCH_BLOCKS] = 0;
    st[KCH_NPEND] = 8;
    st[KCH_NOUT] = 8;
}

// four bytes popped from the END of the output buffer: bytes 4m+3, 4m+2, 4m+1, 4m as a little-endian u32, which is H[m]
__device__ __forceinline__ u32 sch_pop_u32(u32 *st) {
    if (st[KCH_NOUT] == 0) sch_flush(st);
    const u32 m = st[KCH_NOUT] - 1;
    st[KCH_NOUT] = m;
    return st[KCH_OUT + m];
}

// MONTY: field elements as the 4 little-endian bytes of their canonical values; otherwise the words' own bytes (a [u8; 32] digest
// held as 8 words).  Either way the big-endian message word is the byte-swapped value.
template <int F, bool MONTY>
__global__ void sch_observe_kernel(u32 *st, const u32 *vals, size_t n) {
    if (threadIdx.x | blockIdx.x) return;
    if (n == 0) return;
    u32 h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = st[i];
    st[KCH_NOUT] = 0;                                                          // any buffered output is now invalid
    u32 m = st[KCH_NPEND];
    for (size_t j = 0; j < n; j++) {
        st[KCH_PEND + m] = bswap32(MONTY ? from_monty<F>(vals[j]) : vals[j]);
        if (++m == 16) {
            u32 w[16];
#pragma unroll
            for (int i = 0; i < 16; i++) w[i] = st[KCH_PEND + i];
            sha256_compress(h, w);
            st[SCH_BLOCKS]++;
            m = 0;
        }
    }
    st[KCH_NPEND] = m;
#pragma unroll
    for (int i = 0; i < 8; i++) st[i] = h[i];
}

template <int F>
__global__ void sch_sample_kernel(u32 *st, u32 *out, size_t n, bool raw, u32 mask) {
    if (threadIdx.x | blockIdx.x) return;
    for (size_t j = 0; j < n; j++) {
        if (raw) { out[j] = sch_pop_u32(st) & mask; continue; }
        u32 v;
        do { v = sch_pop_u32(st) & 0x7fffffffu; } while (v >= Fp<F>::P);
        out[j] = to_monty<F>(v);
    }
}

// Candidate c is valid iff observe(c); sample_bits(bits) == 0.  Each thread finishes the hash from the midstate: the pending words,
// its candidate and the padding, one or two compressions.  The first sampled u32 is H[7].  best = smallest valid c.
template <int F>
__global__ void __launch_bounds__(128) sch_grind_kernel(const u32 *st, u32 base, u32 count, u32 mask, u32 *best) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const u32 cand = base + t;
    if (cand >= Fp<F>::P) return;
    u32 h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = st[i];
    sch_finish(h, st + KCH_PEND, st[KCH_NPEND], true, bswap32(cand), st[SCH_BLOCKS]);
    if ((h[7] & mask) == 0) atomicMin(best, cand);
}

template <typename Fn> static int32_t field_dispatch(int field, Fn &&fn) {
    if (field == BABY_BEAR) return fn(std::integral_constant<int, BABY_BEAR>());
    return fn(std::integral_constant<int, KOALA_BEAR>());
}

template <typename Fn> static int32_t ch_dispatch(int field, int width, Fn &&fn) {
    if (field == BABY_BEAR && width == 16) return fn(std::integral_constant<int, BABY_BEAR>(), std::integral_constant<int, 16>());
    if (field == BABY_BEAR && width == 24) return fn(std::integral_constant<int, BABY_BEAR>(), std::integral_constant<int, 24>());
    if (field == KOALA_BEAR && width == 16) return fn(std::integral_constant<int, KOALA_BEAR>(), std::integral_constant<int, 16>());
    return fn(std::integral_constant<int, KOALA_BEAR>(), std::integral_constant<int, 24>());
}

static int32_t ch_consts(p3gpu_ctx *ctx, const p3gpu_challenger *ch, const Poseidon2Consts **k) {
    *k = &ctx->p2_host[ch->field][ch->width == 24];
    P3_CHECK((*k)->set, P3GPU_ESTATE, "Poseidon2 constants for field %d width %d not set (p3gpu_poseidon2_set_constants)", ch->field, ch->width);
    return P3GPU_OK;
}

static int32_t challenger_alloc(p3gpu_ctx *ctx, int kind, int field, int width, int rate, p3gpu_challenger **out) {
    p3gpu_challenger *ch = new p3gpu_challenger();
    ch->kind = kind; ch->field = field; ch->width = width; ch->rate = rate;
    if (cudaMalloc(&ch->state, (CH_WORDS + CH_STAGE) * 4) != cudaSuccess) { delete ch; cudaGetLastError(); set_error("cudaMalloc failed"); return P3GPU_ENOMEM; }
    ch->stage = ch->state + CH_WORDS;
    P3_CUDA(cudaMemsetAsync(ch->state, 0, CH_WORDS * 4, ctx->stream));
    *out = ch;
    return P3GPU_OK;
}
int32_t challenger_new(p3gpu_ctx *ctx, int field, int width, int rate, p3gpu_challenger **out) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    P3_CHECK(width == 16 || width == 24, P3GPU_EUNSUPPORTED, "challenger permutation width %d unsupported (16 or 24)", width);
    P3_CHECK(rate > 0 && rate < width && rate <= 24, P3GPU_EINVAL, "challenger rate %d out of range", rate);
    return challenger_alloc(ctx, CH_DUPLEX, field, width, rate, out);
}
// SerializingChallenger32::from_hasher(vec![], Keccak256Hash): an empty input buffer and an empty output buffer (all-zero state)
int32_t challenger_new_keccak256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    return challenger_alloc(ctx, CH_KECCAK256, field, 0, 0, out);
}
// SerializingChallenger32::from_hasher(vec![], Sha256): empty buffers, the midstate at the IV
int32_t challenger_new_sha256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    static const u32 iv[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
    P3_TRY(challenger_alloc(ctx, CH_SHA256, field, 0, 0, out));
    P3_CUDA(cudaMemcpyAsync((*out)->state, iv, sizeof iv, cudaMemcpyHostToDevice, ctx->stream));   // pageable source: staged before return
    return P3GPU_OK;
}
void challenger_free(p3gpu_ctx *ctx, p3gpu_challenger *ch) {
    if (!ch) return;
    cudaStreamSynchronize(ctx->stream);
    cudaFree(ch->state);
    delete ch;
}
int32_t challenger_clone(p3gpu_ctx *ctx, const p3gpu_challenger *src, p3gpu_challenger **out) {
    P3_TRY(challenger_alloc(ctx, src->kind, src->field, src->width, src->rate, out));
    P3_CUDA(cudaMemcpyAsync((*out)->state, src->state, CH_WORDS * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    return P3GPU_OK;
}

static int32_t kch_observe_dev(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *d_vals, size_t n, bool monty) {
    if (n == 0) return P3GPU_OK;
    P3_TRY(field_dispatch(ch->field, [&](auto f) -> int32_t {
        constexpr int F = decltype(f)::value;
        if (ch->kind == CH_SHA256) {
            if (monty) sch_observe_kernel<F, true><<<1, 1, 0, ctx->stream>>>(ch->state, d_vals, n);
            else sch_observe_kernel<F, false><<<1, 1, 0, ctx->stream>>>(ch->state, d_vals, n);
        } else if (monty) {
            kch_observe_kernel<F, true><<<1, 1, 0, ctx->stream>>>(ch->state, d_vals, n);
        } else {
            kch_observe_kernel<F, false><<<1, 1, 0, ctx->stream>>>(ch->state, d_vals, n);
        }
        return P3GPU_OK;
    }));
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}
int32_t challenger_observe_dev(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *d_vals, size_t n) {
    if (ch->kind != CH_DUPLEX) return kch_observe_dev(ctx, ch, d_vals, n, true);
    if (n == 0) return P3GPU_OK;
    const Poseidon2Consts *k;
    P3_TRY(ch_consts(ctx, ch, &k));
    P3_TRY(ch_dispatch(ch->field, ch->width, [&](auto f, auto w) -> int32_t {
        ch_observe_kernel<decltype(f)::value, decltype(w)::value><<<1, 1, 0, ctx->stream>>>(ch->state, ch->rate, d_vals, n, *k);
        return P3GPU_OK;
    }));
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}
int32_t challenger_observe_host(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *h_vals, size_t n) {
    const u32 p = ch->field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    for (size_t i = 0; i < n; i++) P3_CHECK(h_vals[i] < p, P3GPU_EINVAL, "observed value not in canonical Montgomery range");
    for (size_t off = 0; off < n; off += CH_STAGE) {
        const size_t m = std::min<size_t>(CH_STAGE, n - off);
        P3_CUDA(cudaMemcpyAsync(ch->stage, h_vals + off, m * 4, cudaMemcpyHostToDevice, ctx->stream));   // pageable source: staged before return
        P3_TRY(challenger_observe_dev(ctx, ch, ch->stage, m));
    }
    return P3GPU_OK;
}
// Digests as the MMCS commits them: [F; 8] digests are field elements (the duplex handle observes them like any value); a Keccak
// MMCS's [u64; 4] digests are observed as their 32 little-endian bytes (CanObserve<MerkleCap<F, [u64; N]>>), the words' own bytes.
int32_t challenger_observe_digest(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *h_words, size_t n) {
    if (ch->kind == CH_DUPLEX) return challenger_observe_host(ctx, ch, h_words, n);
    for (size_t off = 0; off < n; off += CH_STAGE) {
        const size_t m = std::min<size_t>(CH_STAGE, n - off);
        P3_CUDA(cudaMemcpyAsync(ch->stage, h_words + off, m * 4, cudaMemcpyHostToDevice, ctx->stream));
        P3_TRY(kch_observe_dev(ctx, ch, ch->stage, m, false));
    }
    return P3GPU_OK;
}
static int32_t kch_sample(p3gpu_ctx *ctx, p3gpu_challenger *ch, u32 *h_out, size_t n, bool raw, u32 mask) {
    P3_TRY(field_dispatch(ch->field, [&](auto f) -> int32_t {
        if (ch->kind == CH_SHA256) sch_sample_kernel<decltype(f)::value><<<1, 1, 0, ctx->stream>>>(ch->state, ch->stage, n, raw, mask);
        else kch_sample_kernel<decltype(f)::value><<<1, 1, 0, ctx->stream>>>(ch->state, ch->stage, n, raw, mask);
        return P3GPU_OK;
    }));
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    P3_CUDA(cudaMemcpyAsync(h_out, ch->stage, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}
int32_t challenger_sample(p3gpu_ctx *ctx, p3gpu_challenger *ch, u32 *h_out, size_t n) {
    P3_CHECK(n <= (size_t)CH_STAGE, P3GPU_EINVAL, "too many samples in one call");
    if (n == 0) return P3GPU_OK;
    if (ch->kind != CH_DUPLEX) return kch_sample(ctx, ch, h_out, n, false, 0);
    const Poseidon2Consts *k;
    P3_TRY(ch_consts(ctx, ch, &k));
    P3_TRY(ch_dispatch(ch->field, ch->width, [&](auto f, auto w) -> int32_t {
        ch_sample_kernel<decltype(f)::value, decltype(w)::value><<<1, 1, 0, ctx->stream>>>(ch->state, ch->rate, ch->stage, n, *k);
        return P3GPU_OK;
    }));
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    P3_CUDA(cudaMemcpyAsync(h_out, ch->stage, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}
// CanSampleBits: the duplex challenger masks the canonical value of a sampled field element (duplex_challenger.rs:270-283); the
// serializing challenger masks the raw u32 of 4 popped bytes (serializing_challenger.rs sample_bits).  Both need 2^bits < p.
int32_t challenger_sample_bits(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, size_t n, u32 *h_out) {
    const u32 p = ch->field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    P3_CHECK(bits < 32 && (1ull << bits) < p, P3GPU_EINVAL, "sample_bits(%u): 2^bits must be below the field order", bits);
    P3_CHECK(n <= (size_t)CH_STAGE, P3GPU_EINVAL, "too many samples in one call");
    if (n == 0) return P3GPU_OK;
    if (ch->kind != CH_DUPLEX) return kch_sample(ctx, ch, h_out, n, true, (1u << bits) - 1u);
    P3_TRY(challenger_sample(ctx, ch, h_out, n));
    for (size_t i = 0; i < n; i++)
        h_out[i] = (ch->field == BABY_BEAR ? from_monty<BABY_BEAR>(h_out[i]) : from_monty<KOALA_BEAR>(h_out[i])) & (u32)((1ull << bits) - 1);
    return P3GPU_OK;
}
static int32_t kch_grind(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, u32 *witness_monty) {
    const u32 p = ch->field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    u32 *best = ch->stage + CH_STAGE - 1;
    const u32 mask = (1u << bits) - 1u, batch = 1u << std::min(22u, bits + 3);
    u32 found = 0xffffffffu;
    for (u64 base = 0; base < p && found == 0xffffffffu; base += batch) {
        P3_CUDA(cudaMemsetAsync(best, 0xff, 4, ctx->stream));
        P3_TRY(field_dispatch(ch->field, [&](auto f) -> int32_t {
            if (ch->kind == CH_SHA256) sch_grind_kernel<decltype(f)::value><<<(batch + 127) / 128, 128, 0, ctx->stream>>>(ch->state, (u32)base, batch, mask, best);
            else kch_grind_kernel<decltype(f)::value><<<(batch + 127) / 128, 128, 0, ctx->stream>>>(ch->state, (u32)base, batch, mask, best);
            return P3GPU_OK;
        }));
        ctx->launches++;
        P3_CUDA(cudaGetLastError());
        P3_CUDA(cudaMemcpyAsync(&found, best, 4, cudaMemcpyDeviceToHost, ctx->stream));
        P3_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    P3_CHECK(found != 0xffffffffu, P3GPU_EINVAL, "failed to find proof-of-work witness");
    const u32 wm = ch->field == BABY_BEAR ? to_monty<BABY_BEAR>(found) : to_monty<KOALA_BEAR>(found);
    P3_TRY(challenger_observe_host(ctx, ch, &wm, 1));
    u32 s = 1;
    P3_TRY(kch_sample(ctx, ch, &s, 1, true, mask));
    P3_CHECK(s == 0, P3GPU_ECUDA, "proof-of-work witness failed the check");
    *witness_monty = wm;
    return P3GPU_OK;
}
// grind(bits): smallest witness w (canonical integer; returned in Montgomery form) such that observe(w); sample_bits(bits) == 0.
// The witness is observed and the sample consumed, exactly like check_witness (grinding_challenger.rs:226-229).
int32_t challenger_grind(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, u32 *witness_monty) {
    P3_CHECK(bits < 31, P3GPU_EINVAL, "proof-of-work bits %u too large", bits);
    const u32 p = ch->field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    if (bits == 0) { *witness_monty = 0; return P3GPU_OK; }
    if (ch->kind != CH_DUPLEX) return kch_grind(ctx, ch, bits, witness_monty);
    const Poseidon2Consts *k;
    P3_TRY(ch_consts(ctx, ch, &k));
    u32 *best = ch->stage + CH_STAGE - 1;
    const u32 mask = (1u << bits) - 1u, batch = 1u << std::min(20u, bits + 3);
    u32 found = 0xffffffffu;
    for (u64 base = 0; base < p && found == 0xffffffffu; base += batch) {
        P3_CUDA(cudaMemsetAsync(best, 0xff, 4, ctx->stream));
        P3_TRY(ch_dispatch(ch->field, ch->width, [&](auto f, auto w) -> int32_t {
            ch_grind_kernel<decltype(f)::value, decltype(w)::value><<<(batch + 127) / 128, 128, 0, ctx->stream>>>(ch->state, ch->rate, (u32)base, batch, mask, best, *k);
            return P3GPU_OK;
        }));
        ctx->launches++;
        P3_CUDA(cudaGetLastError());
        P3_CUDA(cudaMemcpyAsync(&found, best, 4, cudaMemcpyDeviceToHost, ctx->stream));
        P3_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    P3_CHECK(found != 0xffffffffu, P3GPU_EINVAL, "failed to find proof-of-work witness");
    const u32 wm = ch->field == BABY_BEAR ? to_monty<BABY_BEAR>(found) : to_monty<KOALA_BEAR>(found);
    P3_TRY(challenger_observe_host(ctx, ch, &wm, 1));
    u32 s = 0;
    P3_TRY(challenger_sample(ctx, ch, &s, 1));
    const u32 canon = ch->field == BABY_BEAR ? from_monty<BABY_BEAR>(s) : from_monty<KOALA_BEAR>(s);
    P3_CHECK((canon & mask) == 0, P3GPU_ECUDA, "proof-of-work witness failed the check");
    *witness_monty = wm;
    return P3GPU_OK;
}

}  // namespace p3
