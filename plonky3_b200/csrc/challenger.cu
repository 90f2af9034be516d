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
// The other two kinds of handle are SerializingChallenger32<F, HashChallenger<u8, H, 32>> (challenger/src/
// serializing_challenger.rs, hash_challenger.rs) over H = Keccak256Hash, the transcript of the Keccak configuration
// (examples/src/types.rs:19-35), and over H = Sha256 (sha256/src/lib.rs), the transcript of the SHA-256 configurations
// (keccak-air/examples/prove_baby_bear_sha256*.rs).  Their state machine is written once in hash_core.cuh, generic over a policy per
// hash (Keccak256Policy, Sha256Policy), so that the host tests run the same code; here it gets one observe, one sample and one
// grind kernel, templated on the field and the policy.
struct p3gpu_challenger {
    int kind;           // CH_DUPLEX, CH_KECCAK256 or CH_SHA256
    int field, width, rate;
    p3::u32 *state;     // device, duplex: [0, width) sponge state | [32, 32+rate) input buffer | [64, 64+rate) output buffer | [96] n_in | [97] n_out
                        //         byte transcripts: the TR_WORDS words laid out in hash_core.cuh
    p3::u32 *stage;     // device staging for host observes / samples (4096 words)
};

namespace p3 {

constexpr int CH_DUPLEX = 0, CH_KECCAK256 = 1, CH_SHA256 = 2;
constexpr int CH_IN = 32, CH_OUT = 64, CH_NIN = 96, CH_NOUT = 97, CH_WORDS = 128, CH_STAGE = 4096;
static_assert(TR_WORDS <= CH_WORDS, "a byte transcript's state fits the state buffer");

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

// ---- SerializingChallenger32<F, HashChallenger<u8, H, 32>>: the state machine of hash_core.cuh, H = Keccak256Policy or
// Sha256Policy ------------------------------------------------------------------------------------------------------------------
template <int F, class H, bool MONTY>
__global__ void tr_observe_kernel(u32 *st, const u32 *vals, size_t n) {
    if (threadIdx.x | blockIdx.x) return;
    transcript_observe<H, F, MONTY>(st, vals, n);
}

template <int F, class H>
__global__ void tr_sample_kernel(u32 *st, u32 *out, size_t n, bool raw, u32 mask) {
    if (threadIdx.x | blockIdx.x) return;
    transcript_sample<H, F>(st, out, n, raw, mask);
}

// Every thread finishes the hash from the midstate for its candidate (one or two Keccak-f or SHA-256 compressions); best = smallest
// valid candidate
template <int F, class H>
__global__ void __launch_bounds__(128) tr_grind_kernel(const u32 *st, u32 base, u32 count, u32 mask, u32 *best) {
    const u32 t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const u32 cand = base + t;
    if (cand >= Fp<F>::P) return;
    if (transcript_is_witness<H>(st, cand, mask)) atomicMin(best, cand);
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

// a byte transcript's field and hash policy as types
template <typename Fn> static int32_t tr_dispatch(const p3gpu_challenger *ch, Fn &&fn) {
    return field_dispatch(ch->field, [&](auto f) -> int32_t {
        if (ch->kind == CH_SHA256) return fn(f, Sha256Policy());
        return fn(f, Keccak256Policy());
    });
}

static u32 field_order(int field) { return field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P; }

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
// SerializingChallenger32::from_hasher(vec![], H): empty buffers, the hash's running state at its start
template <class H> static int32_t tr_new(p3gpu_ctx *ctx, int kind, int field, p3gpu_challenger **out) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    u32 st[TR_WORDS] = {};
    H::init(st);
    P3_TRY(challenger_alloc(ctx, kind, field, 0, 0, out));
    P3_CUDA(cudaMemcpyAsync((*out)->state, st, sizeof st, cudaMemcpyHostToDevice, ctx->stream));   // pageable source: staged before return
    return P3GPU_OK;
}
int32_t challenger_new_keccak256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out) { return tr_new<Keccak256Policy>(ctx, CH_KECCAK256, field, out); }
int32_t challenger_new_sha256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out) { return tr_new<Sha256Policy>(ctx, CH_SHA256, field, out); }
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

// One observe launch over n device words.  monty = false (words observed as their own bytes) only for the byte transcripts.
static int32_t observe_launch(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *d_vals, size_t n, bool monty) {
    if (n == 0) return P3GPU_OK;
    if (ch->kind == CH_DUPLEX) {
        const Poseidon2Consts *k;
        P3_TRY(ch_consts(ctx, ch, &k));
        P3_TRY(ch_dispatch(ch->field, ch->width, [&](auto f, auto w) -> int32_t {
            ch_observe_kernel<decltype(f)::value, decltype(w)::value><<<1, 1, 0, ctx->stream>>>(ch->state, ch->rate, d_vals, n, *k);
            return P3GPU_OK;
        }));
    } else {
        P3_TRY(tr_dispatch(ch, [&](auto f, auto h) -> int32_t {
            constexpr int F = decltype(f)::value;
            if (monty) tr_observe_kernel<F, decltype(h), true><<<1, 1, 0, ctx->stream>>>(ch->state, d_vals, n);
            else tr_observe_kernel<F, decltype(h), false><<<1, 1, 0, ctx->stream>>>(ch->state, d_vals, n);
            return P3GPU_OK;
        }));
    }
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}
static int32_t observe_staged(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *h_vals, size_t n, bool monty) {
    for (size_t off = 0; off < n; off += CH_STAGE) {
        const size_t m = std::min<size_t>(CH_STAGE, n - off);
        P3_CUDA(cudaMemcpyAsync(ch->stage, h_vals + off, m * 4, cudaMemcpyHostToDevice, ctx->stream));   // pageable source: staged before return
        P3_TRY(observe_launch(ctx, ch, ch->stage, m, monty));
    }
    return P3GPU_OK;
}
int32_t challenger_observe_dev(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *d_vals, size_t n) {
    return observe_launch(ctx, ch, d_vals, n, true);
}
int32_t challenger_observe_host(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *h_vals, size_t n) {
    const u32 p = field_order(ch->field);
    for (size_t i = 0; i < n; i++) P3_CHECK(h_vals[i] < p, P3GPU_EINVAL, "observed value not in canonical Montgomery range");
    return observe_staged(ctx, ch, h_vals, n, true);
}
// Digests as the MMCS commits them: [F; 8] digests are field elements (the duplex handle observes them like any value); a Keccak
// or SHA-256 MMCS's [u64; 4] or [u8; 32] digests are observed as their 32 bytes (CanObserve<MerkleCap<F, [u64; 4] | [u8; 32]>>),
// the words' own little-endian bytes.
int32_t challenger_observe_digest(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *h_words, size_t n) {
    if (ch->kind == CH_DUPLEX) return challenger_observe_host(ctx, ch, h_words, n);
    return observe_staged(ctx, ch, h_words, n, false);
}

// One sample launch into the staging buffer, copied back.  raw: the byte transcripts' CanSampleBits, the u32 of 4 popped bytes AND
// mask.
static int32_t sample_launch(p3gpu_ctx *ctx, p3gpu_challenger *ch, u32 *h_out, size_t n, bool raw, u32 mask) {
    if (ch->kind == CH_DUPLEX) {
        const Poseidon2Consts *k;
        P3_TRY(ch_consts(ctx, ch, &k));
        P3_TRY(ch_dispatch(ch->field, ch->width, [&](auto f, auto w) -> int32_t {
            ch_sample_kernel<decltype(f)::value, decltype(w)::value><<<1, 1, 0, ctx->stream>>>(ch->state, ch->rate, ch->stage, n, *k);
            return P3GPU_OK;
        }));
    } else {
        P3_TRY(tr_dispatch(ch, [&](auto f, auto h) -> int32_t {
            tr_sample_kernel<decltype(f)::value, decltype(h)><<<1, 1, 0, ctx->stream>>>(ch->state, ch->stage, n, raw, mask);
            return P3GPU_OK;
        }));
    }
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    P3_CUDA(cudaMemcpyAsync(h_out, ch->stage, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}
int32_t challenger_sample(p3gpu_ctx *ctx, p3gpu_challenger *ch, u32 *h_out, size_t n) {
    P3_CHECK(n <= (size_t)CH_STAGE, P3GPU_EINVAL, "too many samples in one call");
    if (n == 0) return P3GPU_OK;
    return sample_launch(ctx, ch, h_out, n, false, 0);
}
// CanSampleBits: the duplex challenger masks the canonical value of a sampled field element (duplex_challenger.rs:270-283); the
// serializing challenger masks the raw u32 of 4 popped bytes (serializing_challenger.rs sample_bits).  Both need 2^bits < p.
int32_t challenger_sample_bits(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, size_t n, u32 *h_out) {
    P3_CHECK(bits < 32 && (1ull << bits) < field_order(ch->field), P3GPU_EINVAL, "sample_bits(%u): 2^bits must be below the field order", bits);
    P3_CHECK(n <= (size_t)CH_STAGE, P3GPU_EINVAL, "too many samples in one call");
    if (n == 0) return P3GPU_OK;
    const u32 mask = (1u << bits) - 1u;
    P3_TRY(sample_launch(ctx, ch, h_out, n, ch->kind != CH_DUPLEX, mask));
    if (ch->kind == CH_DUPLEX)
        for (size_t i = 0; i < n; i++) h_out[i] = (ch->field == BABY_BEAR ? from_monty<BABY_BEAR>(h_out[i]) : from_monty<KOALA_BEAR>(h_out[i])) & mask;
    return P3GPU_OK;
}

// grind(bits): smallest witness w (canonical integer; returned in Montgomery form) such that observe(w); sample_bits(bits) == 0.
// Batches of candidates are searched in order until one holds a witness; the witness is then observed and the sample consumed,
// exactly like check_witness (grinding_challenger.rs:226-229).
int32_t challenger_grind(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, u32 *witness_monty) {
    P3_CHECK(bits < 31, P3GPU_EINVAL, "proof-of-work bits %u too large", bits);
    if (bits == 0) { *witness_monty = 0; return P3GPU_OK; }
    const Poseidon2Consts *k = nullptr;
    if (ch->kind == CH_DUPLEX) P3_TRY(ch_consts(ctx, ch, &k));
    const u32 p = field_order(ch->field), mask = (1u << bits) - 1u;
    const u32 batch = 1u << std::min(ch->kind == CH_DUPLEX ? 20u : 22u, bits + 3), grid = (batch + 127) / 128;
    u32 *best = ch->stage + CH_STAGE - 1;
    u32 found = 0xffffffffu;
    for (u64 base = 0; base < p && found == 0xffffffffu; base += batch) {
        P3_CUDA(cudaMemsetAsync(best, 0xff, 4, ctx->stream));
        if (ch->kind == CH_DUPLEX) {
            P3_TRY(ch_dispatch(ch->field, ch->width, [&](auto f, auto w) -> int32_t {
                ch_grind_kernel<decltype(f)::value, decltype(w)::value><<<grid, 128, 0, ctx->stream>>>(ch->state, ch->rate, (u32)base, batch, mask, best, *k);
                return P3GPU_OK;
            }));
        } else {
            P3_TRY(tr_dispatch(ch, [&](auto f, auto h) -> int32_t {
                tr_grind_kernel<decltype(f)::value, decltype(h)><<<grid, 128, 0, ctx->stream>>>(ch->state, (u32)base, batch, mask, best);
                return P3GPU_OK;
            }));
        }
        ctx->launches++;
        P3_CUDA(cudaGetLastError());
        P3_CUDA(cudaMemcpyAsync(&found, best, 4, cudaMemcpyDeviceToHost, ctx->stream));
        P3_CUDA(cudaStreamSynchronize(ctx->stream));
    }
    P3_CHECK(found != 0xffffffffu, P3GPU_EINVAL, "failed to find proof-of-work witness");
    const u32 wm = ch->field == BABY_BEAR ? to_monty<BABY_BEAR>(found) : to_monty<KOALA_BEAR>(found);
    P3_TRY(challenger_observe_host(ctx, ch, &wm, 1));
    u32 s = 1;
    P3_TRY(challenger_sample_bits(ctx, ch, bits, 1, &s));
    P3_CHECK(s == 0, P3GPU_ECUDA, "proof-of-work witness failed the check");
    *witness_monty = wm;
    return P3GPU_OK;
}

}  // namespace p3
