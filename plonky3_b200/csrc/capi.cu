// extern "C" surface of libp3gpu (include/p3gpu.h): context, memory plumbing, host-pointer wrappers and the
// PCS-level drivers (TwoAdicFriPcs::commit, fri commit phase) built from the NTT / hash / fold kernels.
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.h"

namespace p3 {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}

static int32_t grow(void **buf, size_t *cap, size_t bytes, cudaStream_t s) {
    if (*cap >= bytes) return P3GPU_OK;
    if (*buf) { P3_CUDA(cudaStreamSynchronize(s)); P3_CUDA(cudaFree(*buf)); *buf = nullptr; *cap = 0; }
    cudaError_t e = cudaMalloc(buf, bytes);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); cudaGetLastError(); return P3GPU_ENOMEM; }
    *cap = bytes;
    return P3GPU_OK;
}
int32_t ctx_scratch(p3gpu_ctx *ctx, size_t bytes, void **out) {
    P3_TRY(grow(&ctx->scratch, &ctx->scratch_bytes, bytes, ctx->stream));
    *out = ctx->scratch;
    return P3GPU_OK;
}
int32_t ctx_scratch2(p3gpu_ctx *ctx, size_t bytes, void **out) {
    P3_TRY(grow(&ctx->scratch2, &ctx->scratch2_bytes, bytes, ctx->stream));
    *out = ctx->scratch2;
    return P3GPU_OK;
}
int32_t ctx_lde_tiles(p3gpu_ctx *ctx, size_t bytes, void **out) {
    P3_TRY(grow(&ctx->lde_tiles, &ctx->lde_tiles_bytes, bytes, ctx->stream));
    *out = ctx->lde_tiles;
    return P3GPU_OK;
}

int32_t ctx_pool(p3gpu_ctx *ctx, int slot, size_t bytes, void **out) {
    P3_TRY(grow(&ctx->pool[slot], &ctx->pool_bytes[slot], bytes ? bytes : 1, ctx->stream));
    *out = ctx->pool[slot];
    return P3GPU_OK;
}

int32_t ctx_leaf_table(p3gpu_ctx *ctx, size_t bytes, void **out) {
    P3_TRY(grow(&ctx->leaf_table, &ctx->leaf_table_bytes, bytes, ctx->stream));
    *out = ctx->leaf_table;
    return P3GPU_OK;
}

struct DevBuf {  // RAII device allocation for the host-pointer wrappers
    void *p = nullptr;
    ~DevBuf() { if (p) cudaFree(p); }
    int32_t alloc(size_t bytes) {
        cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); cudaGetLastError(); p = nullptr; return P3GPU_ENOMEM; }
        return P3GPU_OK;
    }
};

}  // namespace p3

using namespace p3;

extern "C" {

const char *p3gpu_last_error(void) { return g_err; }

int32_t p3gpu_ctx_create(int device, p3gpu_ctx **out) {
    P3_CHECK(out != nullptr, P3GPU_EINVAL, "ctx_create: null output pointer");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        set_error("no CUDA device available (%s): libp3gpu has no CPU fallback", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        cudaGetLastError();
        return P3GPU_ECUDA;
    }
    P3_CHECK(device >= 0 && device < n, P3GPU_EINVAL, "device %d out of range (0..%d)", device, n - 1);
    P3_CUDA(cudaSetDevice(device));
    p3gpu_ctx *ctx = new p3gpu_ctx();
    ctx->device = device;
    memset(ctx->p2_host, 0, sizeof ctx->p2_host);
    cudaDeviceProp prop;
    P3_CUDA(cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    P3_CUDA(cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking));
    P3_CUDA(cudaEventCreateWithFlags(&ctx->switch_event, cudaEventDisableTiming));
    ctx->stream = ctx->own_stream;
    if (const char *mb = getenv("P3GPU_TWIDDLE_CACHE_MB")) ctx->twiddle_cap_bytes = (size_t)strtoull(mb, nullptr, 10) << 20;
    *out = ctx;
    return P3GPU_OK;
}

void p3gpu_ctx_destroy(p3gpu_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (auto &kv : ctx->twiddles) cudaFree(kv.second.ptr);
    if (ctx->leaf_table) cudaFree(ctx->leaf_table);
    if (ctx->switch_event) cudaEventDestroy(ctx->switch_event);
    if (ctx->h2d_stream) { cudaStreamDestroy(ctx->h2d_stream); cudaStreamDestroy(ctx->d2h_stream); cudaEventDestroy(ctx->ev_start); }
    for (int b = 0; b < 2; b++) {
        if (ctx->ev_h2d[b]) { cudaEventDestroy(ctx->ev_h2d[b]); cudaEventDestroy(ctx->ev_comp[b]); cudaEventDestroy(ctx->ev_d2h[b]); }
        if (ctx->chunk_in[b]) cudaFree(ctx->chunk_in[b]);
        if (ctx->chunk_out[b]) cudaFree(ctx->chunk_out[b]);
    }
    for (int f = 0; f < 2; f++) if (ctx->fold_table[f]) cudaFree(ctx->fold_table[f]);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->scratch2) cudaFree(ctx->scratch2);
    if (ctx->lde_tiles) cudaFree(ctx->lde_tiles);
    if (ctx->p1_consts) cudaFree(ctx->p1_consts);
    for (int i = 0; i < 4; i++) if (ctx->pool[i]) cudaFree(ctx->pool[i]);
    if (ctx->xchg_stream) cudaStreamDestroy(ctx->xchg_stream);
    for (int q = 0; q < 16; q++) if (ctx->dma_stream[q]) { cudaStreamDestroy(ctx->dma_stream[q]); cudaEventDestroy(ctx->dma_done[q]); }
    for (int b = 0; b < 2; b++) {
        if (ctx->ev_stage_full[b]) { cudaEventDestroy(ctx->ev_stage_full[b]); cudaEventDestroy(ctx->ev_stage_free[b]); }
        if (ctx->stage_buf[b]) cudaFree(ctx->stage_buf[b]);
    }
    if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
    delete ctx;
}

// The context's scratch buffers, pools, fold tables and twiddle heaps are shared by all of its calls and ordered only by the stream
// they were used on.  When the caller moves the context to another stream, work already queued on the old stream (which may
// still read or write those buffers, or be generating a twiddle heap) must finish before anything on the new stream touches
// them: record an event on the old stream and make the new one wait for it.
static int32_t switch_stream(p3gpu_ctx *ctx, cudaStream_t s) {
    if (s == ctx->stream) return P3GPU_OK;
    P3_CUDA(cudaEventRecord(ctx->switch_event, ctx->stream));
    P3_CUDA(cudaStreamWaitEvent(s, ctx->switch_event, 0));
    ctx->stream = s;
    return P3GPU_OK;
}
int32_t p3gpu_ctx_set_stream(p3gpu_ctx *ctx, void *cuda_stream) {
    P3_ENTER(ctx);
    return switch_stream(ctx, (cudaStream_t)cuda_stream);  // NULL is the legacy default stream (what torch uses by default)
}
int32_t p3gpu_ctx_use_own_stream(p3gpu_ctx *ctx) {
    P3_ENTER(ctx);
    return switch_stream(ctx, ctx->own_stream);
}
int32_t p3gpu_ctx_sync(p3gpu_ctx *ctx) {
    P3_ENTER(ctx);
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}
uint64_t p3gpu_launch_count(const p3gpu_ctx *ctx) { return ctx ? ctx->launches : 0; }

int32_t p3gpu_malloc(p3gpu_ctx *ctx, size_t bytes, void **dptr) {
    P3_ENTER(ctx);
    P3_CHECK(dptr, P3GPU_EINVAL, "null argument");
    cudaError_t e = cudaMalloc(dptr, bytes ? bytes : 1);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); cudaGetLastError(); return P3GPU_ENOMEM; }
    return P3GPU_OK;
}
int32_t p3gpu_free(p3gpu_ctx *ctx, void *dptr) {
    P3_ENTER(ctx);
    if (dptr) { P3_CUDA(cudaStreamSynchronize(ctx->stream)); P3_CUDA(cudaFree(dptr)); }
    return P3GPU_OK;
}
int32_t p3gpu_memcpy_h2d(p3gpu_ctx *ctx, void *dst, const void *src, size_t bytes) {
    P3_ENTER(ctx);
    P3_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
    return P3GPU_OK;
}
int32_t p3gpu_memcpy_d2h(p3gpu_ctx *ctx, void *dst, const void *src, size_t bytes) {
    P3_ENTER(ctx);
    P3_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}
int32_t p3gpu_host_register(void *ptr, size_t bytes) {
    P3_CUDA(cudaHostRegister(ptr, bytes, cudaHostRegisterDefault));
    return P3GPU_OK;
}
int32_t p3gpu_host_unregister(void *ptr) {
    P3_CUDA(cudaHostUnregister(ptr));
    return P3GPU_OK;
}

// ---- TwoAdicSubgroupDft ------------------------------------------------------------------------
int32_t p3gpu_dft_batch_dev(p3gpu_ctx *ctx, int field, int kind, const uint32_t *d_in, uint32_t *d_out, size_t h, size_t w,
                            uint32_t shift) {
    P3_ENTER(ctx);
    P3_CHECK(d_in && d_out, P3GPU_EINVAL, "null argument");
    return ntt_dft_batch(ctx, field, kind, d_in, d_out, h, w, shift);
}
int32_t p3gpu_dft_batch(p3gpu_ctx *ctx, int field, int kind, uint32_t *h_inout, size_t h, size_t w, uint32_t shift) {
    P3_ENTER(ctx);
    P3_CHECK(h_inout, P3GPU_EINVAL, "null argument");
    void *buf = nullptr;
    P3_TRY(ctx_pool(ctx, 0, h * w * 4, &buf));
    P3_CUDA(cudaMemcpyAsync(buf, h_inout, h * w * 4, cudaMemcpyHostToDevice, ctx->stream));
    P3_TRY(ntt_dft_batch(ctx, field, kind, (const u32 *)buf, (u32 *)buf, h, w, shift));
    P3_CUDA(cudaMemcpyAsync(h_inout, buf, h * w * 4, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}
int32_t p3gpu_coset_lde_batch_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_in, size_t h, size_t w, unsigned added_bits,
                                  uint32_t shift, uint32_t *d_out, int bitrev_rows) {
    P3_ENTER(ctx);
    P3_CHECK(d_in && d_out, P3GPU_EINVAL, "null argument");
    return ntt_coset_lde(ctx, field, d_in, h, w, added_bits, shift, d_out, bitrev_rows);
}
int32_t p3gpu_lde_coefficients_dev(p3gpu_ctx *ctx, int field, uint32_t *d_trace, size_t h, size_t w) {
    P3_ENTER(ctx);
    P3_CHECK(d_trace, P3GPU_EINVAL, "null argument");
    return ntt_lde_coefficients(ctx, field, d_trace, h, w);
}
int32_t p3gpu_lde_coset_block_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_coeffs, size_t h, size_t w, unsigned added_bits,
                                  uint32_t shift, size_t coset, uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_coeffs && d_out, P3GPU_EINVAL, "null argument");
    return ntt_lde_coset_block(ctx, field, d_coeffs, h, w, added_bits, shift, coset, d_out);
}
// ---- host-pointer pipeline ------------------------------------------------------------------------
// A host-pointer call is PCIe-bound (config 2: 419 MB in and 839 MB out over PCIe against milliseconds of compute).  The matrix
// is cut into column chunks (every column is an independent polynomial) and the three stages run on three streams:
//     H2D(chunk i+1)  ||  LDE(chunk i)  ||  D2H(chunk i-1)
// PCIe is full duplex, so one call approaches max(H2D, D2H) + one chunk instead of H2D + compute + D2H.  Chunks travel as 2-D
// copies (row segments of the chunk's width at the caller's pitch) into compact double-buffered device buffers.
static int32_t pipeline_setup(p3gpu_ctx *ctx) {
    if (ctx->h2d_stream) return P3GPU_OK;
    P3_CUDA(cudaStreamCreateWithFlags(&ctx->h2d_stream, cudaStreamNonBlocking));
    P3_CUDA(cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking));
    for (int b = 0; b < 2; b++) {
        P3_CUDA(cudaEventCreateWithFlags(&ctx->ev_h2d[b], cudaEventDisableTiming));
        P3_CUDA(cudaEventCreateWithFlags(&ctx->ev_comp[b], cudaEventDisableTiming));
        P3_CUDA(cudaEventCreateWithFlags(&ctx->ev_d2h[b], cudaEventDisableTiming));
    }
    P3_CUDA(cudaEventCreateWithFlags(&ctx->ev_start, cudaEventDisableTiming));
    return P3GPU_OK;
}
// column chunk boundaries in units of 8 columns (the tiled LDE path needs width % 4 == 0 and >= 8; sectors stay aligned)
static std::vector<size_t> column_chunks(size_t w, size_t n_chunks) {
    std::vector<size_t> b{0};
    const size_t units = w / 8;
    if (n_chunks > units) n_chunks = units;
    if (n_chunks <= 1 || w % 4 != 0) { b.push_back(w); return b; }
    // the FIRST chunk takes the remainder, so the grow-only scratch buffers are sized by the first LDE call and never
    // reallocated (a reallocation synchronises the stream) in the middle of the pipeline
    for (size_t c = 1; c <= n_chunks; c++) b.push_back(c == n_chunks ? w : w - (units * (n_chunks - c) / n_chunks) * 8);
    return b;
}
// Chunks of the round-trip pipeline (p3gpu_coset_lde_batch).  Default 1 = strictly serial contiguous copies: the copy engines
// move 2-D chunks with narrow (96-192 byte) row segments of a 400-byte-pitch matrix markedly slower than contiguous copies,
// which eats the overlap for the 2^20 x 100 LDE (tools/pcie_probe.py measures both on a given host).  Wide matrices
// (>= 512-byte row segments per chunk) do profit: set P3GPU_E2E_CHUNKS.
static size_t host_chunk_count(size_t bytes_in, size_t dflt) {
    if (bytes_in < ((size_t)16 << 20)) return 1;          // small calls: latency, not bandwidth
    const char *e = getenv("P3GPU_E2E_CHUNKS");
    const long v = e ? atol(e) : (long)dflt;
    return (size_t)(v < 1 ? 1 : v > 64 ? 64 : v);
}

int32_t p3gpu_coset_lde_batch(p3gpu_ctx *ctx, int field, const uint32_t *h_in, size_t h, size_t w, unsigned added_bits,
                              uint32_t shift, uint32_t *h_out, int bitrev_rows) {
    P3_ENTER(ctx);
    P3_CHECK(h_in && h_out, P3GPU_EINVAL, "null argument");
    P3_CHECK(added_bits <= 8, P3GPU_EINVAL, "added_bits %u too large", added_bits);
    const size_t nin = h * w * 4, nout = nin << added_bits, H = h << added_bits;
    const std::vector<size_t> cb = column_chunks(w, bitrev_rows && h >= 4096 ? host_chunk_count(nin, 1) : 1);
    if (cb.size() == 2) {                                   // one chunk: strictly serial H2D -> LDE -> D2H on the context's stream
        void *in = nullptr, *out = nullptr;
        P3_TRY(ctx_pool(ctx, 0, nin, &in));
        P3_TRY(ctx_pool(ctx, 1, nout, &out));
        P3_CUDA(cudaMemcpyAsync(in, h_in, nin, cudaMemcpyHostToDevice, ctx->stream));
        P3_TRY(ntt_coset_lde(ctx, field, (const u32 *)in, h, w, added_bits, shift, (u32 *)out, bitrev_rows));
        P3_CUDA(cudaMemcpyAsync(h_out, out, nout, cudaMemcpyDeviceToHost, ctx->stream));
        P3_CUDA(cudaStreamSynchronize(ctx->stream));
        return P3GPU_OK;
    }
    P3_TRY(pipeline_setup(ctx));
    size_t wmax = 0;
    for (size_t c = 0; c + 1 < cb.size(); c++) wmax = std::max(wmax, cb[c + 1] - cb[c]);
    for (int b = 0; b < 2; b++) {
        P3_TRY(grow(&ctx->chunk_in[b], &ctx->chunk_in_bytes[b], h * wmax * 4, ctx->stream));
        P3_TRY(grow(&ctx->chunk_out[b], &ctx->chunk_out_bytes[b], H * wmax * 4, ctx->stream));
    }
    // earlier work of this context (other entry points on ctx->stream) owns the chunk buffers until it is done
    P3_CUDA(cudaEventRecord(ctx->ev_start, ctx->stream));
    P3_CUDA(cudaStreamWaitEvent(ctx->h2d_stream, ctx->ev_start, 0));
    P3_CUDA(cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_start, 0));
    for (size_t c = 0; c + 1 < cb.size(); c++) {
        const int b = (int)(c & 1);
        const size_t c0 = cb[c], wc = cb[c + 1] - c0;
        if (c >= 2) P3_CUDA(cudaStreamWaitEvent(ctx->h2d_stream, ctx->ev_comp[b], 0));          // chunk c-2 has consumed chunk_in[b]
        P3_CUDA(cudaMemcpy2DAsync(ctx->chunk_in[b], wc * 4, h_in + c0, w * 4, wc * 4, h, cudaMemcpyHostToDevice, ctx->h2d_stream));
        P3_CUDA(cudaEventRecord(ctx->ev_h2d[b], ctx->h2d_stream));
        P3_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[b], 0));
        if (c >= 2) P3_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_d2h[b], 0));              // chunk c-2 has left chunk_out[b]
        P3_TRY(ntt_coset_lde(ctx, field, (const u32 *)ctx->chunk_in[b], h, wc, added_bits, shift, (u32 *)ctx->chunk_out[b], bitrev_rows));
        P3_CUDA(cudaEventRecord(ctx->ev_comp[b], ctx->stream));
        P3_CUDA(cudaStreamWaitEvent(ctx->d2h_stream, ctx->ev_comp[b], 0));
        P3_CUDA(cudaMemcpy2DAsync(h_out + c0, w * 4, ctx->chunk_out[b], wc * 4, wc * 4, H, cudaMemcpyDeviceToHost, ctx->d2h_stream));
        P3_CUDA(cudaEventRecord(ctx->ev_d2h[b], ctx->d2h_stream));
    }
    P3_CUDA(cudaStreamSynchronize(ctx->d2h_stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}

// ---- hashing -----------------------------------------------------------------------------------
int32_t p3gpu_poseidon2_set_constants(p3gpu_ctx *ctx, int field, int width, const uint32_t *rc_initial, const uint32_t *rc_terminal,
                                      const uint32_t *rc_internal, int rounds_p) {
    P3_ENTER(ctx);
    P3_CHECK(rc_initial && rc_terminal && rc_internal, P3GPU_EINVAL, "null argument");
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    P3_CHECK(width == 16 || width == 24, P3GPU_EUNSUPPORTED, "Poseidon2 width %d unsupported (16 or 24)", width);
    P3_CHECK(rounds_p >= 1 && rounds_p <= 32, P3GPU_EINVAL, "rounds_p %d out of range", rounds_p);
    const uint32_t p = field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    Poseidon2Consts &k = ctx->p2_host[field][width == 24];
    memset(&k, 0, sizeof k);
    for (int i = 0; i < 4 * width; i++) {
        P3_CHECK(rc_initial[i] < p && rc_terminal[i] < p, P3GPU_EINVAL, "round constant not in canonical Montgomery range");
        k.rc_ext[i] = rc_initial[i]; k.rc_ext[4 * width + i] = rc_terminal[i];
    }
    for (int i = 0; i < rounds_p; i++) {
        P3_CHECK(rc_internal[i] < p, P3GPU_EINVAL, "round constant not in canonical Montgomery range");
        k.rc_int[i] = rc_internal[i];
    }
    k.rounds_p = rounds_p; k.width = width; k.set = 1;
    return P3GPU_OK;
}
int32_t p3gpu_poseidon2_permute_dev(p3gpu_ctx *ctx, int field, int width, uint32_t *d_states, size_t n) {
    P3_ENTER(ctx);
    P3_CHECK(d_states, P3GPU_EINVAL, "null argument");
    return hash_poseidon2_permute(ctx, field, width, d_states, n);
}
int32_t p3gpu_keccak_f_dev(p3gpu_ctx *ctx, uint64_t *d_states, size_t n) {
    P3_ENTER(ctx);
    P3_CHECK(d_states, P3GPU_EINVAL, "null argument");
    return hash_keccak_f(ctx, d_states, n);
}

size_t p3gpu_merkle_total_digests(size_t max_height) {
    auto pad = [](size_t raw) { return raw <= 1 ? raw : (raw + 1) / 2 * 2; };
    size_t len = pad(max_height), tot = len;
    while (len > 1) { len = pad(len / 2); tot += len; }
    return tot;
}
int32_t p3gpu_merkle_commit_dev(p3gpu_ctx *ctx, int field, int hash, size_t n_mats, const uint32_t *const *d_mats,
                                const size_t *heights, const size_t *widths, uint32_t *d_layers, size_t *layer_lens,
                                size_t *n_layers) {
    P3_ENTER(ctx);
    P3_CHECK(d_mats && heights && widths && d_layers && layer_lens && n_layers, P3GPU_EINVAL, "null argument");
    return hash_merkle_commit(ctx, field, hash, n_mats, d_mats, heights, widths, d_layers, layer_lens, n_layers);
}
int32_t p3gpu_merkle_commit(p3gpu_ctx *ctx, int field, int hash, size_t n_mats, const uint32_t *const *h_mats,
                            const size_t *heights, const size_t *widths, uint32_t *h_layers, size_t *layer_lens,
                            size_t *n_layers) {
    P3_ENTER(ctx);
    P3_CHECK(h_mats && heights && widths && h_layers && layer_lens && n_layers, P3GPU_EINVAL, "null argument");
    P3_CHECK(n_mats >= 1 && n_mats <= (1u << 20), P3GPU_EINVAL, "No matrices given?");
    // one pooled arena for all matrices + one for the digest layers (grow-only context buffers: no cudaMalloc/cudaFree per call)
    std::vector<size_t> offs(n_mats);
    size_t arena = 0, max_h = 0;
    for (size_t i = 0; i < n_mats; i++) {
        offs[i] = arena;
        arena += (heights[i] * widths[i] * 4 + 255) & ~(size_t)255;
        if (heights[i] > max_h) max_h = heights[i];
    }
    void *mats = nullptr, *layers = nullptr;
    P3_TRY(ctx_pool(ctx, 0, arena, &mats));
    const size_t tot = p3gpu_merkle_total_digests(max_h);
    P3_TRY(ctx_pool(ctx, 1, tot * 32, &layers));
    std::vector<const u32 *> ptrs(n_mats);
    for (size_t i = 0; i < n_mats; i++) {
        const size_t bytes = heights[i] * widths[i] * 4;
        ptrs[i] = reinterpret_cast<const u32 *>((unsigned char *)mats + offs[i]);
        if (bytes) P3_CUDA(cudaMemcpyAsync((void *)ptrs[i], h_mats[i], bytes, cudaMemcpyHostToDevice, ctx->stream));
    }
    P3_TRY(hash_merkle_commit(ctx, field, hash, n_mats, ptrs.data(), heights, widths, (u32 *)layers, layer_lens, n_layers));
    P3_CUDA(cudaMemcpyAsync(h_layers, layers, tot * 32, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}

int32_t p3gpu_merkle_from_digests_dev(p3gpu_ctx *ctx, int field, int hash, const uint32_t *d_digests, size_t n, uint32_t *d_layers,
                                      size_t *layer_lens, size_t *n_layers) {
    P3_ENTER(ctx);
    P3_CHECK(d_digests && d_layers && layer_lens && n_layers, P3GPU_EINVAL, "null argument");
    return hash_merkle_from_digests(ctx, field, hash, d_digests, n, d_layers, layer_lens, n_layers);
}

// ---- FRI ---------------------------------------------------------------------------------------
int32_t p3gpu_fri_fold_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_in, size_t rows, unsigned log_arity, const uint32_t beta[4],
                           uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_in && d_out && beta, P3GPU_EINVAL, "null argument");
    return fri_fold(ctx, field, d_in, rows, log_arity, beta, d_out);
}
int32_t p3gpu_fri_fold(p3gpu_ctx *ctx, int field, const uint32_t *h_in, size_t rows, unsigned log_arity, const uint32_t beta[4],
                       uint32_t *h_out) {
    P3_ENTER(ctx);
    P3_CHECK(h_in && h_out && beta, P3GPU_EINVAL, "null argument");
    P3_CHECK(log_arity >= 1 && log_arity <= 4, P3GPU_EINVAL, "log_arity %u out of range 1..4", log_arity);
    void *in = nullptr, *out = nullptr;
    const size_t nin = (rows << log_arity) * 16;
    P3_TRY(ctx_pool(ctx, 0, nin, &in));
    P3_TRY(ctx_pool(ctx, 1, rows * 16, &out));
    P3_CUDA(cudaMemcpyAsync(in, h_in, nin, cudaMemcpyHostToDevice, ctx->stream));
    P3_TRY(fri_fold(ctx, field, (const u32 *)in, rows, log_arity, beta, (u32 *)out));
    P3_CUDA(cudaMemcpyAsync(h_out, out, rows * 16, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}

int32_t p3gpu_ef_axpy_dev(p3gpu_ctx *ctx, int field, uint32_t *d_acc, const uint32_t *d_x, size_t n, const uint32_t s[4]) {
    P3_ENTER(ctx);
    P3_CHECK(d_acc && d_x && s, P3GPU_EINVAL, "null argument");
    return fri_ef_axpy(ctx, field, d_acc, d_x, n, s);
}

// fri/src/config.rs:180-207 with a single input vector (next_input_log_height = None)
static unsigned log_arity_for_round(unsigned log_cur, unsigned log_final, unsigned max_log_arity) {
    const unsigned m = log_cur - log_final;
    return m < max_log_arity ? m : max_log_arity;
}

int32_t p3gpu_fri_commit_phase_dev(p3gpu_ctx *ctx, int field, int hash, uint32_t *d_vec, size_t len, unsigned log_blowup,
                                   unsigned log_final_poly_len, unsigned max_log_arity, unsigned cap_height, const uint32_t *betas,
                                   size_t n_betas, uint32_t *h_caps, size_t *cap_lens, unsigned *log_arities, size_t *n_rounds,
                                   uint32_t *h_final) {
    P3_ENTER(ctx);
    P3_CHECK(d_vec && betas && h_caps && cap_lens && log_arities && n_rounds && h_final, P3GPU_EINVAL, "null argument");
    P3_CHECK(is_pow2(len), P3GPU_EINVAL, "commit phase: length %zu is not a power of two", len);
    P3_CHECK(max_log_arity >= 1 && max_log_arity <= 4, P3GPU_EINVAL, "max_log_arity must be in 1..4 to guarantee folding progress");
    const unsigned log_final = log_blowup + log_final_poly_len;
    // digest layers of the largest round + ping-pong buffer for the folded vector
    const unsigned la0 = log2_floor(len) > log_final ? log_arity_for_round(log2_floor(len), log_final, max_log_arity) : 1;
    void *layers = nullptr, *pong = nullptr;
    P3_TRY(ctx_pool(ctx, 2, p3gpu_merkle_total_digests(len >> la0) * 32, &layers));
    P3_TRY(ctx_pool(ctx, 3, (len >> la0) * 16 + 16, &pong));
    u32 *cur = d_vec, *other = (u32 *)pong;
    size_t cur_len = len, round = 0, cap_off = 0;
    while (cur_len > ((size_t)1 << log_final)) {
        P3_CHECK(round < n_betas, P3GPU_EINVAL, "commit phase: %zu betas supplied, more rounds needed", n_betas);
        const unsigned la = log_arity_for_round(log2_floor(cur_len), log_final, max_log_arity);
        const size_t rows = cur_len >> la, width = ((size_t)4) << la;  // ExtensionMmcs: EF4 -> 4 base columns
        const u32 *mats[1] = {cur};
        size_t lens[65], nl = 0;
        P3_TRY(hash_merkle_commit(ctx, field, hash, 1, mats, &rows, &width, (u32 *)layers, lens, &nl));
        // cap(min(cap_height, layers-1)): mmcs/batch.rs:56-62, merkle_tree.rs:198-217
        const size_t eff = cap_height < nl - 1 ? cap_height : nl - 1;
        size_t off = 0;
        for (size_t k = 0; k + 1 + eff < nl; k++) off += lens[k];
        const size_t cl = std::min((size_t)1 << eff, lens[nl - 1 - eff]);
        P3_CUDA(cudaMemcpyAsync(h_caps + cap_off * 8, (u32 *)layers + off * 8, cl * 32, cudaMemcpyDeviceToHost, ctx->stream));
        cap_lens[round] = cl; cap_off += cl; log_arities[round] = la;
        P3_TRY(fri_fold(ctx, field, cur, rows, la, betas + 4 * round, other));
        std::swap(cur, other);
        cur_len = rows; round++;
    }
    P3_CUDA(cudaMemcpyAsync(h_final, cur, cur_len * 16, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    *n_rounds = round;
    return P3GPU_OK;
}

// ---- Pcs::open (pre-FRI part) ------------------------------------------------------------------
int32_t p3gpu_open_inv_denoms_dev(p3gpu_ctx *ctx, int field, unsigned log_height, const uint32_t z[4], const uint32_t *zinv,
                                  uint32_t *d_inv_denoms, uint32_t *d_adjusted) {
    P3_ENTER(ctx);
    P3_CHECK(z && d_inv_denoms, P3GPU_EINVAL, "null argument");
    return open_inv_denoms(ctx, field, log_height, z, zinv, d_inv_denoms, d_adjusted);
}
int32_t p3gpu_columnwise_dot_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_mat, size_t h, size_t w, const uint32_t *d_vec_ef,
                                 const uint32_t *scale, uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_mat && d_vec_ef && d_out, P3GPU_EINVAL, "null argument");
    return open_columnwise_dot(ctx, field, d_mat, h, w, d_vec_ef, d_out, scale);
}
int32_t p3gpu_rowwise_dot_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_mat, size_t h, size_t w, const uint32_t alpha[4], uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_mat && alpha && d_out, P3GPU_EINVAL, "null argument");
    return open_rowwise_dot(ctx, field, d_mat, h, w, alpha, d_out);
}
int32_t p3gpu_open_reduce_dev(p3gpu_ctx *ctx, int field, uint32_t *d_ro, const uint32_t *d_r, const uint32_t *d_inv_denoms, size_t h,
                              const uint32_t coeff[4], const uint32_t yred[4]) {
    P3_ENTER(ctx);
    P3_CHECK(d_ro && d_r && d_inv_denoms && coeff && yred, P3GPU_EINVAL, "null argument");
    return open_reduce(ctx, field, d_ro, d_r, d_inv_denoms, h, coeff, yred);
}

// ---- Poseidon2 AIR: trace generation + quotient (SURVEY 8f ranks 2-3) --------------------------------
int32_t p3gpu_p2air_set_constants(p3gpu_ctx *ctx, int field, const uint32_t *beginning_full, const uint32_t *partial, int rounds_p,
                                  const uint32_t *ending_full) {
    P3_ENTER(ctx);
    P3_CHECK(beginning_full && partial && ending_full, P3GPU_EINVAL, "null argument");
    return air_set_constants(ctx, field, beginning_full, partial, rounds_p, ending_full);
}
size_t p3gpu_p2air_columns(int rounds_p) { return 144 + (size_t)rounds_p; }
size_t p3gpu_p2air_field_columns(int field, int rounds_p) { return air_columns(field, rounds_p); }
int32_t p3gpu_p2air_generate_trace_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_inputs, size_t n_perms, uint32_t *d_trace) {
    P3_ENTER(ctx);
    P3_CHECK(d_inputs && d_trace, P3GPU_EINVAL, "null argument");
    return air_generate_trace(ctx, field, d_inputs, n_perms, d_trace);
}
int32_t p3gpu_p2air_quotient_dev(p3gpu_ctx *ctx, int field, int vector_len, const uint32_t *d_lde, unsigned log_lde_height, unsigned log_trace_height,
                                 const uint32_t alpha[4], uint32_t *d_quotient) {
    P3_ENTER(ctx);
    P3_CHECK(d_lde && alpha && d_quotient, P3GPU_EINVAL, "null argument");
    return air_quotient(ctx, field, vector_len, d_lde, log_lde_height, log_trace_height, alpha, d_quotient);
}
int32_t p3gpu_p2air_generate_trace_cols_dev(p3gpu_ctx *ctx, int field, int vector_len, const uint32_t *d_inputs, size_t n_perms, size_t col0,
                                            size_t col1, uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_TRY(air_sharded_field(field));
    P3_CHECK(d_inputs && (d_out || col0 == col1), P3GPU_EINVAL, "null argument");
    return air_generate_trace_cols(ctx, field, vector_len, d_inputs, n_perms, col0, col1, d_out);
}

// ---- Keccak-f AIR: trace generation + quotient (keccak_air.cu) ----------------------------------------
int32_t p3gpu_keccak_air_generate_trace_dev(p3gpu_ctx *ctx, int field, const uint64_t *d_inputs, size_t n_hashes, uint32_t *d_trace) {
    P3_ENTER(ctx);
    P3_CHECK((d_inputs || n_hashes == 0) && d_trace, P3GPU_EINVAL, "null argument");
    P3_CHECK(reinterpret_cast<uintptr_t>(d_inputs) % 8 == 0 && reinterpret_cast<uintptr_t>(d_trace) % 4 == 0, P3GPU_EINVAL,
             "Keccak AIR trace: misaligned buffer");
    return keccak_air_generate(ctx, field, d_inputs, n_hashes, d_trace);
}
int32_t p3gpu_keccak_air_quotient_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_lde, unsigned log_lde_height, unsigned log_trace_height,
                                      const uint32_t alpha[4], uint32_t *d_quotient) {
    P3_ENTER(ctx);
    P3_CHECK(d_lde && alpha && d_quotient, P3GPU_EINVAL, "null argument");
    return keccak_air_quotient(ctx, field, d_lde, log_lde_height, log_trace_height, alpha, d_quotient);
}

// ---- Blake3 AIR: trace generation + quotient (blake3_air.cu) ------------------------------------------
int32_t p3gpu_blake3_air_generate_trace_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_inputs, size_t n_hashes, uint32_t *d_trace) {
    P3_ENTER(ctx);
    P3_CHECK(d_inputs && d_trace, P3GPU_EINVAL, "null argument");
    P3_CHECK(reinterpret_cast<uintptr_t>(d_inputs) % 4 == 0 && reinterpret_cast<uintptr_t>(d_trace) % 4 == 0, P3GPU_EINVAL,
             "Blake3 AIR trace: misaligned buffer");
    return blake3_air_generate(ctx, field, d_inputs, n_hashes, d_trace);
}
int32_t p3gpu_blake3_air_quotient_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_lde, unsigned log_lde_height, unsigned log_trace_height,
                                      const uint32_t alpha[4], uint32_t *d_quotient) {
    P3_ENTER(ctx);
    P3_CHECK(d_lde && alpha && d_quotient, P3GPU_EINVAL, "null argument");
    return blake3_air_quotient(ctx, field, d_lde, log_lde_height, log_trace_height, alpha, d_quotient);
}
int32_t p3gpu_blake3_air_generate_trace_cols_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_inputs, size_t n_hashes, size_t col0, size_t col1,
                                                 uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_inputs && (d_out || col0 == col1), P3GPU_EINVAL, "null argument");
    P3_CHECK(reinterpret_cast<uintptr_t>(d_inputs) % 4 == 0 && reinterpret_cast<uintptr_t>(d_out) % 4 == 0, P3GPU_EINVAL,
             "Blake3 AIR trace: misaligned buffer");
    return blake3_air_generate_cols(ctx, field, d_inputs, n_hashes, col0, col1, d_out);
}

// ---- SHA-256 AIR: trace generation + quotient (sha256_air.cu) -----------------------------------------
int32_t p3gpu_sha256_air_generate_trace_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_inputs, size_t n_hashes, uint32_t *d_trace) {
    P3_ENTER(ctx);
    P3_CHECK(d_inputs && d_trace, P3GPU_EINVAL, "null argument");
    P3_CHECK(reinterpret_cast<uintptr_t>(d_inputs) % 4 == 0 && reinterpret_cast<uintptr_t>(d_trace) % 4 == 0, P3GPU_EINVAL,
             "SHA-256 AIR trace: misaligned buffer");
    return sha256_air_generate(ctx, field, d_inputs, n_hashes, d_trace);
}
int32_t p3gpu_sha256_air_quotient_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_lde, unsigned log_lde_height, unsigned log_trace_height,
                                      const uint32_t alpha[4], uint32_t *d_quotient) {
    P3_ENTER(ctx);
    P3_CHECK(d_lde && alpha && d_quotient, P3GPU_EINVAL, "null argument");
    return sha256_air_quotient(ctx, field, d_lde, log_lde_height, log_trace_height, alpha, d_quotient);
}
int32_t p3gpu_sha256_air_generate_trace_cols_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_inputs, size_t n_hashes, size_t col0, size_t col1,
                                                 uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_inputs && (d_out || col0 == col1), P3GPU_EINVAL, "null argument");
    P3_CHECK(reinterpret_cast<uintptr_t>(d_inputs) % 4 == 0 && reinterpret_cast<uintptr_t>(d_out) % 4 == 0, P3GPU_EINVAL,
             "SHA-256 AIR trace: misaligned buffer");
    return sha256_air_generate_cols(ctx, field, d_inputs, n_hashes, col0, col1, d_out);
}

// ---- Poseidon1 AIR: constants, trace generation + quotient (poseidon1_air.cu) -------------------------------
int32_t p3gpu_p1air_set_constants(p3gpu_ctx *ctx, int field, const uint32_t *initial_full, const uint32_t *terminal_full,
                                  const uint32_t *mds_circ_col, const uint32_t *first_round_constants, const uint32_t *m_i,
                                  const uint32_t *partial_rc, const uint32_t *sparse_first_row, const uint32_t *v, int rounds_p) {
    P3_ENTER(ctx);
    P3_CHECK(initial_full && terminal_full && mds_circ_col && first_round_constants && m_i && sparse_first_row && v && (partial_rc || rounds_p == 1),
             P3GPU_EINVAL, "null argument");
    return p1air_set_constants(ctx, field, initial_full, terminal_full, mds_circ_col, first_round_constants, m_i, partial_rc, sparse_first_row, v,
                               rounds_p);
}
size_t p3gpu_p1air_columns(int field, int rounds_p) { return p1air_columns(field, rounds_p); }
int32_t p3gpu_p1air_generate_trace_dev(p3gpu_ctx *ctx, int field, const uint32_t *d_inputs, size_t n_perms, uint32_t *d_trace) {
    P3_ENTER(ctx);
    P3_CHECK(d_inputs && d_trace, P3GPU_EINVAL, "null argument");
    return p1air_generate(ctx, field, d_inputs, n_perms, d_trace);
}
int32_t p3gpu_p1air_quotient_dev(p3gpu_ctx *ctx, int field, int vector_len, const uint32_t *d_lde, unsigned log_lde_height, unsigned log_trace_height,
                                 const uint32_t alpha[4], uint32_t *d_quotient) {
    P3_ENTER(ctx);
    P3_CHECK(d_lde && alpha && d_quotient, P3GPU_EINVAL, "null argument");
    return p1air_quotient(ctx, field, vector_len, d_lde, log_lde_height, log_trace_height, alpha, d_quotient);
}
int32_t p3gpu_p1air_generate_trace_cols_dev(p3gpu_ctx *ctx, int field, int vector_len, const uint32_t *d_inputs, size_t n_perms, size_t col0,
                                            size_t col1, uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_inputs && (d_out || col0 == col1), P3GPU_EINVAL, "null argument");
    return p1air_generate_cols(ctx, field, vector_len, d_inputs, n_perms, col0, col1, d_out);
}

// ---- any AIR as a constraint program (air_program.cu) -------------------------------------------------
int32_t p3gpu_air_program_create(p3gpu_ctx *ctx, int field, const p3gpu_air_node *nodes, size_t n_nodes, const uint32_t *constraints,
                                 size_t n_constraints, uint32_t width, uint32_t n_public, p3gpu_air_program **out) {
    P3_ENTER(ctx);
    P3_CHECK(out, P3GPU_EINVAL, "null argument");
    *out = nullptr;
    const p3gpu_air_layout layout = {width, n_public, 0, 0};
    return air_program_create(ctx, field, nodes, n_nodes, constraints, n_constraints, layout, out);
}
int32_t p3gpu_air_program_create_layout(p3gpu_ctx *ctx, int field, const p3gpu_air_node *nodes, size_t n_nodes, const uint32_t *constraints,
                                        size_t n_constraints, const p3gpu_air_layout *layout, p3gpu_air_program **out) {
    P3_ENTER(ctx);
    P3_CHECK(out && layout, P3GPU_EINVAL, "null argument");
    *out = nullptr;
    return air_program_create(ctx, field, nodes, n_nodes, constraints, n_constraints, *layout, out);
}
void p3gpu_air_program_destroy(p3gpu_air_program *prog) { air_program_destroy(prog); }
int32_t p3gpu_air_program_info(const p3gpu_air_program *prog, size_t *n_instructions, size_t *n_slots, size_t *n_constraints) {
    return air_program_info(prog, n_instructions, n_slots, n_constraints);
}
int32_t p3gpu_air_quotient_dev(p3gpu_ctx *ctx, const p3gpu_air_program *prog, const uint32_t *d_lde, unsigned log_lde_height,
                               unsigned log_quotient_size, unsigned log_trace_height, const uint32_t *public_values, const uint32_t alpha[4],
                               uint32_t *d_quotient) {
    P3_ENTER(ctx);
    P3_CHECK(prog && d_lde && alpha && d_quotient, P3GPU_EINVAL, "null argument");
    return air_program_quotient(ctx, prog, d_lde, log_lde_height, nullptr, 0, nullptr, 0, log_quotient_size, log_trace_height, public_values,
                                alpha, d_quotient, false);
}
int32_t p3gpu_air_quotient_layout_dev(p3gpu_ctx *ctx, const p3gpu_air_program *prog, const uint32_t *d_lde, unsigned log_lde_height,
                                      const uint32_t *d_pre_lde, unsigned log_pre_lde_height, const uint32_t *d_periodic,
                                      unsigned log_periodic_rows, unsigned log_quotient_size, unsigned log_trace_height,
                                      const uint32_t *public_values, const uint32_t alpha[4], uint32_t *d_quotient) {
    P3_ENTER(ctx);
    P3_CHECK(prog && d_lde && alpha && d_quotient, P3GPU_EINVAL, "null argument");
    return air_program_quotient(ctx, prog, d_lde, log_lde_height, d_pre_lde, log_pre_lde_height, d_periodic, log_periodic_rows,
                                log_quotient_size, log_trace_height, public_values, alpha, d_quotient, true);
}

int32_t p3gpu_air_check_program_create(p3gpu_ctx *ctx, int field, const p3gpu_air_node *nodes, size_t n_nodes, const uint32_t *constraints,
                                       size_t n_constraints, const p3gpu_air_layout *layout, p3gpu_air_program **out) {
    P3_ENTER(ctx);
    P3_CHECK(out && layout, P3GPU_EINVAL, "null argument");
    *out = nullptr;
    return air_program_create(ctx, field, nodes, n_nodes, constraints, n_constraints, *layout, out, true);
}
int32_t p3gpu_air_check_dev(p3gpu_ctx *ctx, const p3gpu_air_program *prog, const uint32_t *d_trace, size_t height, const uint32_t *d_preprocessed,
                            const uint32_t *d_periodic, size_t periodic_rows, const uint32_t *public_values, uint32_t *d_counts) {
    P3_ENTER(ctx);
    P3_CHECK(prog && d_trace && d_counts, P3GPU_EINVAL, "null argument");
    return air_check(ctx, prog, d_trace, height, d_preprocessed, d_periodic, periodic_rows, public_values, d_counts, nullptr, 0, nullptr, nullptr);
}
int32_t p3gpu_air_check_rows_dev(p3gpu_ctx *ctx, const p3gpu_air_program *prog, const uint32_t *d_trace, size_t height,
                                 const uint32_t *d_preprocessed, const uint32_t *d_periodic, size_t periodic_rows, const uint32_t *public_values,
                                 const uint32_t *d_rows, size_t n_rows, const uint64_t *d_offsets, uint32_t *d_failed) {
    P3_ENTER(ctx);
    P3_CHECK(prog && d_trace && (n_rows == 0 || (d_rows && d_offsets && d_failed)), P3GPU_EINVAL, "null argument");
    return air_check(ctx, prog, d_trace, height, d_preprocessed, d_periodic, periodic_rows, public_values, nullptr, d_rows, n_rows, d_offsets,
                     d_failed);
}

// ---- transcript + query phase (prove driver) ---------------------------------------------------------
int32_t p3gpu_challenger_new(p3gpu_ctx *ctx, int field, int width, int rate, p3gpu_challenger **out) {
    P3_ENTER(ctx);
    P3_CHECK(out, P3GPU_EINVAL, "null argument");
    return challenger_new(ctx, field, width, rate, out);
}
void p3gpu_challenger_free(p3gpu_ctx *ctx, p3gpu_challenger *ch) {
    if (!ctx) return;
    std::lock_guard<std::recursive_mutex> lock(ctx->call_mu);
    cudaSetDevice(ctx->device);
    challenger_free(ctx, ch);
}
int32_t p3gpu_challenger_clone(p3gpu_ctx *ctx, const p3gpu_challenger *src, p3gpu_challenger **out) {
    P3_ENTER(ctx);
    P3_CHECK(src && out, P3GPU_EINVAL, "null argument");
    return challenger_clone(ctx, src, out);
}
int32_t p3gpu_challenger_observe_dev(p3gpu_ctx *ctx, p3gpu_challenger *ch, const uint32_t *d_values, size_t n) {
    P3_ENTER(ctx);
    P3_CHECK(ch && (d_values || n == 0), P3GPU_EINVAL, "null argument");
    return challenger_observe_dev(ctx, ch, d_values, n);
}
int32_t p3gpu_challenger_observe(p3gpu_ctx *ctx, p3gpu_challenger *ch, const uint32_t *h_values, size_t n) {
    P3_ENTER(ctx);
    P3_CHECK(ch && (h_values || n == 0), P3GPU_EINVAL, "null argument");
    return challenger_observe_host(ctx, ch, h_values, n);
}
int32_t p3gpu_challenger_sample(p3gpu_ctx *ctx, p3gpu_challenger *ch, uint32_t *h_out, size_t n) {
    P3_ENTER(ctx);
    P3_CHECK(ch && h_out, P3GPU_EINVAL, "null argument");
    return challenger_sample(ctx, ch, h_out, n);
}
int32_t p3gpu_challenger_grind(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, uint32_t *witness) {
    P3_ENTER(ctx);
    P3_CHECK(ch && witness, P3GPU_EINVAL, "null argument");
    return challenger_grind(ctx, ch, bits, witness);
}
int32_t p3gpu_challenger_new_keccak256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out) {
    P3_ENTER(ctx);
    P3_CHECK(out, P3GPU_EINVAL, "null argument");
    return challenger_new_keccak256(ctx, field, out);
}
int32_t p3gpu_challenger_new_sha256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out) {
    P3_ENTER(ctx);
    P3_CHECK(out, P3GPU_EINVAL, "null argument");
    return challenger_new_sha256(ctx, field, out);
}
int32_t p3gpu_challenger_observe_digest(p3gpu_ctx *ctx, p3gpu_challenger *ch, const uint32_t *h_words, size_t n) {
    P3_ENTER(ctx);
    P3_CHECK(ch && (h_words || n == 0), P3GPU_EINVAL, "null argument");
    return challenger_observe_digest(ctx, ch, h_words, n);
}
int32_t p3gpu_challenger_sample_bits(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, size_t n, uint32_t *h_out) {
    P3_ENTER(ctx);
    P3_CHECK(ch && (h_out || n == 0), P3GPU_EINVAL, "null argument");
    return challenger_sample_bits(ctx, ch, bits, n, h_out);
}
int32_t p3gpu_gather_rows_dev(p3gpu_ctx *ctx, const uint32_t *d_mat, size_t h, size_t w, const uint32_t *h_indices, size_t n, unsigned index_shift,
                              uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_mat && h_indices && d_out, P3GPU_EINVAL, "null argument");
    return query_gather_rows(ctx, d_mat, h, w, h_indices, n, index_shift, d_out);
}
int32_t p3gpu_merkle_paths_dev(p3gpu_ctx *ctx, const uint32_t *d_layers, const size_t *layer_lens, size_t n_layers, size_t path_len,
                               const uint32_t *h_indices, size_t n, unsigned index_shift, uint32_t *d_out) {
    P3_ENTER(ctx);
    P3_CHECK(d_layers && layer_lens && h_indices && d_out, P3GPU_EINVAL, "null argument");
    return query_merkle_paths(ctx, d_layers, layer_lens, n_layers, path_len, h_indices, n, index_shift, d_out);
}

// ---- multi-GPU: CUDA IPC plumbing + the row-sharded commit ---------------------------------------
int32_t p3gpu_ipc_export(p3gpu_ctx *ctx, void *dptr, uint8_t handle[64]) {
    P3_ENTER(ctx);
    P3_CHECK(dptr && handle, P3GPU_EINVAL, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    cudaIpcMemHandle_t h;
    P3_CUDA(cudaIpcGetMemHandle(&h, dptr));
    memcpy(handle, &h, 64);
    return P3GPU_OK;
}
int32_t p3gpu_ipc_import(p3gpu_ctx *ctx, const uint8_t handle[64], void **dptr) {
    P3_ENTER(ctx);
    P3_CHECK(dptr && handle, P3GPU_EINVAL, "null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    P3_CUDA(cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
    return P3GPU_OK;
}
int32_t p3gpu_ipc_close(p3gpu_ctx *ctx, void *dptr) {
    P3_ENTER(ctx);
    if (dptr) { P3_CUDA(cudaStreamSynchronize(ctx->stream)); P3_CUDA(cudaIpcCloseMemHandle(dptr)); }
    return P3GPU_OK;
}
int32_t p3gpu_memset_dev(p3gpu_ctx *ctx, void *dptr, int value, size_t bytes) {
    P3_ENTER(ctx);
    P3_CHECK(dptr, P3GPU_EINVAL, "null argument");
    P3_CUDA(cudaMemsetAsync(dptr, value, bytes, ctx->stream));
    return P3GPU_OK;
}

static int32_t check_group(const p3gpu_peer_group *g, bool need_rows) {
    P3_CHECK(g != nullptr, P3GPU_EINVAL, "null peer group");
    P3_CHECK(g->world >= 1 && g->world <= 16 && (g->world & (g->world - 1)) == 0 && g->rank < g->world, P3GPU_EINVAL,
             "peer group: world %u (power of two <= 16), rank %u", g->world, g->rank);
    for (uint32_t q = 0; q < g->world; q++) {
        P3_CHECK(g->ctrl[q] != nullptr, P3GPU_EINVAL, "peer group: null control block of rank %u", q);
        P3_CHECK(!need_rows || g->rows[q] != nullptr, P3GPU_EINVAL, "peer group: null row block of rank %u", q);
    }
    return P3GPU_OK;
}

int32_t p3gpu_peer_barrier_dev(p3gpu_ctx *ctx, const p3gpu_peer_group *grp, uint32_t epoch) {
    P3_ENTER(ctx);
    P3_TRY(check_group(grp, false));
    return peer_barrier(ctx, grp->world, grp->rank, grp->ctrl, epoch, grp->timeout_s > 0 ? grp->timeout_s : 20.0);
}

int32_t p3gpu_peer_allgather_dev(p3gpu_ctx *ctx, const p3gpu_peer_group *grp, size_t table_offset_bytes, const uint32_t *d_src, size_t words) {
    P3_ENTER(ctx);
    P3_TRY(check_group(grp, false));
    P3_CHECK(d_src != nullptr && table_offset_bytes % 4 == 0, P3GPU_EINVAL, "bad argument");
    P3_CHECK(P3GPU_PEER_CTRL_USER + table_offset_bytes + (size_t)grp->world * words * 4 <= P3GPU_PEER_CTRL_BYTES, P3GPU_EINVAL,
             "all-gather table does not fit the control block");
    void *tabs[16];
    for (uint32_t q = 0; q < grp->world; q++) tabs[q] = (unsigned char *)grp->ctrl[q] + P3GPU_PEER_CTRL_USER + table_offset_bytes;
    return peer_allgather(ctx, grp->world, grp->rank, tabs, d_src, words);
}

int32_t p3gpu_coset_lde_batch_sharded_dev(p3gpu_ctx *ctx, int field, const p3gpu_peer_group *grp, const uint32_t *d_in, size_t h, size_t w_local,
                                          unsigned added_bits, uint32_t shift, size_t w_total, size_t col_off) {
    P3_ENTER(ctx);
    P3_TRY(check_group(grp, true));
    P3_CHECK(d_in != nullptr || w_local == 0, P3GPU_EINVAL, "null argument");
    return ntt_coset_lde_sharded(ctx, field, d_in, h, w_local, added_bits, shift, grp->world, grp->rows, w_total, col_off);
}

size_t p3gpu_shard_chunk_bounds(size_t w_local, size_t *bounds, size_t max_bounds) {
    const std::vector<size_t> cb = shard_chunk_bounds(w_local);
    for (size_t i = 0; i < cb.size() && i < max_bounds; i++) bounds[i] = cb[i];
    return cb.size();
}

int32_t p3gpu_shard_col_segments(uint32_t world, const size_t *col_starts, size_t rows, size_t *segs, size_t max_segs, size_t *n_segs) {
    P3_CHECK(col_starts && n_segs && (segs || max_segs == 0), P3GPU_EINVAL, "null argument");
    std::vector<size_t> s;
    P3_TRY(shard_col_segments(world, col_starts, rows, s));
    *n_segs = s.size() / 3;
    P3_CHECK(*n_segs <= max_segs, P3GPU_EINVAL, "%zu column segments, room for %zu", *n_segs, max_segs);
    for (size_t i = 0; i < s.size(); i++) segs[i] = s[i];
    return P3GPU_OK;
}

int32_t p3gpu_peer_exchange_dev(p3gpu_ctx *ctx, const p3gpu_peer_group *grp, uint32_t *epoch, void *const *bufs, const uint32_t *d_src, size_t words) {
    P3_ENTER(ctx);
    P3_TRY(check_group(grp, false));
    P3_CHECK(epoch && bufs && (d_src || words == 0), P3GPU_EINVAL, "null argument");
    for (uint32_t q = 0; q < grp->world; q++) P3_CHECK(bufs[q] != nullptr, P3GPU_EINVAL, "null exchange buffer of rank %u", q);
    const double tmo = grp->timeout_s > 0 ? grp->timeout_s : 20.0;
    // nobody overwrites a slot before every rank has finished reading the previous exchange out of its buffer
    P3_TRY(peer_barrier(ctx, grp->world, grp->rank, grp->ctrl, ++*epoch, tmo));
    if (words)
        for (uint32_t q = 0; q < grp->world; q++)     // copy-engine peer copies, stream-ordered before the closing barrier
            P3_CUDA(cudaMemcpyAsync((u32 *)bufs[q] + (size_t)grp->rank * words, d_src, words * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    return peer_barrier(ctx, grp->world, grp->rank, grp->ctrl, ++*epoch, tmo);
}

int32_t p3gpu_p2air_quotient_sharded_dev(p3gpu_ctx *ctx, int field, int vector_len, const p3gpu_peer_group *grp, const size_t *col_starts,
                                         unsigned log_lde_height, unsigned log_trace_height, const uint32_t alpha[4], uint32_t *d_quotient_slice) {
    P3_ENTER(ctx);
    P3_TRY(air_sharded_field(field));
    P3_TRY(check_group(grp, true));
    P3_CHECK(col_starts && alpha && d_quotient_slice, P3GPU_EINVAL, "null argument");
    return air_quotient_sharded(ctx, field, vector_len, grp->world, grp->rank, grp->rows[grp->rank], col_starts, log_lde_height, log_trace_height,
                                alpha, d_quotient_slice);
}

// the Blake3, SHA-256 and Poseidon1 AIRs' sharded quotients: air_hand_quotient's sharded mode on my row block
static int32_t hand_shard(const p3gpu_peer_group *grp, const size_t *col_starts, const uint32_t *alpha, const uint32_t *d_q, AirHandShard &sh) {
    P3_TRY(check_group(grp, true));
    P3_CHECK(col_starts && alpha && d_q, P3GPU_EINVAL, "null argument");
    sh = AirHandShard{grp->world, grp->rank, col_starts, 0};
    return P3GPU_OK;
}
int32_t p3gpu_blake3_air_quotient_sharded_dev(p3gpu_ctx *ctx, int field, const p3gpu_peer_group *grp, const size_t *col_starts,
                                              unsigned log_lde_height, unsigned log_trace_height, const uint32_t alpha[4],
                                              uint32_t *d_quotient_slice) {
    P3_ENTER(ctx);
    AirHandShard sh;
    P3_TRY(hand_shard(grp, col_starts, alpha, d_quotient_slice, sh));
    return blake3_air_quotient_sharded(ctx, field, sh, grp->rows[grp->rank], log_lde_height, log_trace_height, alpha, d_quotient_slice);
}
int32_t p3gpu_sha256_air_quotient_sharded_dev(p3gpu_ctx *ctx, int field, const p3gpu_peer_group *grp, const size_t *col_starts,
                                              unsigned log_lde_height, unsigned log_trace_height, const uint32_t alpha[4],
                                              uint32_t *d_quotient_slice) {
    P3_ENTER(ctx);
    AirHandShard sh;
    P3_TRY(hand_shard(grp, col_starts, alpha, d_quotient_slice, sh));
    return sha256_air_quotient_sharded(ctx, field, sh, grp->rows[grp->rank], log_lde_height, log_trace_height, alpha, d_quotient_slice);
}
int32_t p3gpu_p1air_quotient_sharded_dev(p3gpu_ctx *ctx, int field, int vector_len, const p3gpu_peer_group *grp, const size_t *col_starts,
                                         unsigned log_lde_height, unsigned log_trace_height, const uint32_t alpha[4],
                                         uint32_t *d_quotient_slice) {
    P3_ENTER(ctx);
    AirHandShard sh;
    P3_TRY(hand_shard(grp, col_starts, alpha, d_quotient_slice, sh));
    return p1air_quotient_sharded(ctx, field, vector_len, sh, grp->rows[grp->rank], log_lde_height, log_trace_height, alpha, d_quotient_slice);
}

int32_t p3gpu_air_quotient_sharded_dev(p3gpu_ctx *ctx, const p3gpu_air_program *prog, const p3gpu_peer_group *grp, const size_t *col_starts,
                                       const uint32_t *d_periodic, unsigned log_periodic_rows, unsigned log_lde_height, unsigned log_trace_height,
                                       const uint32_t *public_values, const uint32_t alpha[4], uint32_t *d_quotient_slice) {
    P3_ENTER(ctx);
    P3_TRY(check_group(grp, true));
    P3_CHECK(prog && col_starts && alpha && d_quotient_slice, P3GPU_EINVAL, "null argument");
    return air_program_quotient_sharded(ctx, prog, grp->world, grp->rank, grp->rows, col_starts, d_periodic, log_periodic_rows, log_lde_height,
                                        log_trace_height, public_values, alpha, d_quotient_slice);
}

// TwoAdicFriPcs::commit of ONE trace whose columns are sharded over the ranks, bit-identical to the single-GPU commitment.
int32_t p3gpu_commit_sharded_dev(p3gpu_ctx *ctx, int field, int hash, const p3gpu_peer_group *grp, uint32_t *epoch, const uint32_t *d_evals_local,
                                 size_t h, const size_t *col_starts, unsigned log_blowup, unsigned cap_height,
                                 uint32_t *d_sub_layers, size_t *layer_lens, size_t *n_layers, uint32_t *h_cap, size_t *cap_len, float *phase_ms) {
    P3_ENTER(ctx);
    P3_TRY(check_group(grp, true));
    P3_CHECK(epoch && col_starts && d_sub_layers && layer_lens && n_layers && h_cap && cap_len, P3GPU_EINVAL, "null argument");
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    const unsigned world = grp->world, rank = grp->rank, log_g = log2_floor(world);
    for (unsigned g = 0; g < world; g++) P3_CHECK(col_starts[g] <= col_starts[g + 1], P3GPU_EINVAL, "column blocks must be ordered");
    P3_CHECK(col_starts[0] == 0, P3GPU_EINVAL, "column blocks must start at 0");
    const size_t w_total = col_starts[world], col_off = col_starts[rank], w_local = col_starts[rank + 1] - col_off;
    P3_CHECK(d_evals_local || w_local == 0, P3GPU_EINVAL, "null argument");
    const size_t H = h << log_blowup, rows = H / world;
    const double tmo = grp->timeout_s > 0 ? grp->timeout_s : 20.0;
    struct PhaseEvents {                             // destroyed on every return path
        cudaEvent_t e[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
        ~PhaseEvents() { for (auto &x : e) if (x) cudaEventDestroy(x); }
    } pe;
    cudaEvent_t *ev = pe.e;
    if (phase_ms) for (auto &e : pe.e) P3_CUDA(cudaEventCreate(&e));
    auto mark = [&](int k) -> int32_t { if (phase_ms) P3_CUDA(cudaEventRecord(ev[k], ctx->stream)); return P3GPU_OK; };
    // the row blocks may still be read by the previous commit's hashing on some rank: nobody starts overwriting them before
    // every rank has entered this call
    P3_TRY(peer_barrier(ctx, world, rank, grp->ctrl, ++*epoch, tmo));
    P3_TRY(mark(0));
    // 1) LDE of my column block, exchanged chunk by chunk into the row blocks of the ranks that will hash those rows.  With more
    //    than one rank the row blocks are CHUNK-MAJOR: every (source rank, column chunk) is its own contiguous (rows x chunk width)
    //    matrix at element offset rows * (first column of the chunk), so the exchange is a plain contiguous copy at link rate and
    //    the leaf sponge runs over the chunk matrices in column order — the same digest as over the dense row (merkle_tree.rs:312-316)
    const int chunk_major = world > 1;
    const u32 shift = field == BABY_BEAR ? to_monty<BABY_BEAR>(Fp<BABY_BEAR>::GEN) : to_monty<KOALA_BEAR>(Fp<KOALA_BEAR>::GEN);
    P3_TRY(ntt_coset_lde_sharded(ctx, field, d_evals_local, h, w_local, log_blowup, shift, world, grp->rows, w_total, col_off, chunk_major));
    P3_TRY(mark(1));
    // 2) all ranks' chunks have landed in my row block
    P3_TRY(peer_barrier(ctx, world, rank, grp->ctrl, ++*epoch, tmo));
    P3_TRY(mark(2));
    // 3) my rows are a complete sub-tree of the global tree (rows of the bit-reversed LDE, merkle_tree.rs:268-338)
    std::vector<const u32 *> mats;
    std::vector<size_t> hs, ws;
    if (!chunk_major) { mats.push_back(grp->rows[rank]); hs.push_back(rows); ws.push_back(w_total); }
    else
        for (unsigned g = 0; g < world; g++) {
            const std::vector<size_t> cb = shard_chunk_bounds(col_starts[g + 1] - col_starts[g]);
            for (size_t c = 0; c + 1 < cb.size(); c++) {
                if (cb[c + 1] == cb[c]) continue;
                mats.push_back(grp->rows[rank] + rows * (col_starts[g] + cb[c]));
                hs.push_back(rows); ws.push_back(cb[c + 1] - cb[c]);
            }
        }
    P3_TRY(hash_merkle_commit(ctx, field, hash, mats.size(), mats.data(), hs.data(), ws.data(), d_sub_layers, layer_lens, n_layers));
    P3_TRY(mark(3));
    // 4) exchange the slice of every sub-tree that the cap (or the levels above the sub-tree roots) is made of
    const size_t nl = *n_layers;
    const unsigned eff = cap_height > log_g ? std::min<unsigned>(cap_height - log_g, (unsigned)(nl - 1)) : 0;   // level below my sub-tree root
    size_t off = 0;
    for (size_t k = 0; k + 1 + eff < nl; k++) off += layer_lens[k];
    const size_t slice = std::min((size_t)1 << eff, layer_lens[nl - 1 - eff]);          // digests per rank
    P3_CHECK(P3GPU_PEER_CTRL_USER + world * slice * 32 * 3 <= P3GPU_PEER_CTRL_BYTES, P3GPU_EUNSUPPORTED, "cap_height %u too large for the control block", cap_height);
    void *tabs[16];
    for (unsigned q = 0; q < world; q++) tabs[q] = (unsigned char *)grp->ctrl[q] + P3GPU_PEER_CTRL_USER;
    P3_TRY(peer_allgather(ctx, world, rank, tabs, d_sub_layers + off * 8, slice * 8));
    P3_TRY(peer_barrier(ctx, world, rank, grp->ctrl, ++*epoch, tmo));
    u32 *table = (u32 *)tabs[rank];
    if (cap_height >= log_g) {                       // the gathered slices ARE the cap (8 GPUs, cap_height 3: the sub-tree roots)
        *cap_len = world * slice;
        P3_CUDA(cudaMemcpyAsync(h_cap, table, *cap_len * 32, cudaMemcpyDeviceToHost, ctx->stream));
    } else {                                         // compress the top log2(world) levels redundantly on every rank
        u32 *top = table + (size_t)world * 8;        // behind the gathered roots inside the control block's user area
        size_t tl[65], tn = 0;
        P3_TRY(hash_merkle_from_digests(ctx, field, hash, table, world, top, tl, &tn));
        size_t toff = 0;
        for (size_t k = 0; k + 1 + cap_height < tn; k++) toff += tl[k];
        *cap_len = (size_t)1 << cap_height;
        P3_CUDA(cudaMemcpyAsync(h_cap, top + toff * 8, *cap_len * 32, cudaMemcpyDeviceToHost, ctx->stream));
    }
    P3_TRY(mark(4));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    if (phase_ms)
        for (int k = 0; k < 4; k++) P3_CUDA(cudaEventElapsedTime(&phase_ms[k], ev[k], ev[k + 1]));
    return P3GPU_OK;
}

// ---- Pcs::commit -------------------------------------------------------------------------------
int32_t p3gpu_pcs_commit_dev(p3gpu_ctx *ctx, int field, int hash, const uint32_t *d_evals, size_t h, size_t w, unsigned log_blowup,
                             uint32_t *d_lde, uint32_t *d_layers, size_t *layer_lens, size_t *n_layers) {
    P3_ENTER(ctx);
    P3_CHECK(d_evals && d_lde && d_layers && layer_lens && n_layers, P3GPU_EINVAL, "null argument");
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    // shift = GENERATOR / domain.shift() with domain.shift() = 1 (two_adic_pcs.rs:312)
    const u32 shift = field == BABY_BEAR ? to_monty<BABY_BEAR>(Fp<BABY_BEAR>::GEN) : to_monty<KOALA_BEAR>(Fp<KOALA_BEAR>::GEN);
    P3_TRY(ntt_coset_lde(ctx, field, d_evals, h, w, log_blowup, shift, d_lde, 1));
    const u32 *mats[1] = {d_lde};
    const size_t lh = h << log_blowup;
    return hash_merkle_commit(ctx, field, hash, 1, mats, &lh, &w, d_layers, layer_lens, n_layers);
}


// Pcs::commit with the trace in HOST memory and everything it produces resident on the device (SURVEY section 7 hard part 1:
// the realistic integration point of a GpuFriPcs): the trace crosses PCIe once, in column chunks whose H2D copies overlap
// the LDE of the previous chunk (written straight into the resident LDE at its column offset); only the cap comes back.
int32_t p3gpu_pcs_commit(p3gpu_ctx *ctx, int field, int hash, const uint32_t *h_evals, size_t h, size_t w, unsigned log_blowup,
                         unsigned cap_height, uint32_t *d_lde, uint32_t *d_layers, size_t *layer_lens, size_t *n_layers,
                         uint32_t *h_cap, size_t *cap_len) {
    P3_ENTER(ctx);
    P3_CHECK(h_evals && d_lde && d_layers && layer_lens && n_layers && h_cap && cap_len, P3GPU_EINVAL, "null argument");
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    const u32 shift = field == BABY_BEAR ? to_monty<BABY_BEAR>(Fp<BABY_BEAR>::GEN) : to_monty<KOALA_BEAR>(Fp<KOALA_BEAR>::GEN);
    const size_t nin = h * w * 4;
    const std::vector<size_t> cb = column_chunks(w, h >= 4096 ? std::max<size_t>(host_chunk_count(nin, 4), nin >> 29) : 1);   // <= 512 MB per chunk
    if (cb.size() == 2) {
        void *in = nullptr;
        P3_TRY(ctx_pool(ctx, 0, nin, &in));
        P3_CUDA(cudaMemcpyAsync(in, h_evals, nin, cudaMemcpyHostToDevice, ctx->stream));
        P3_TRY(ntt_coset_lde(ctx, field, (const u32 *)in, h, w, log_blowup, shift, d_lde, 1));
    } else {
        P3_TRY(pipeline_setup(ctx));
        size_t wmax = 0;
        for (size_t c = 0; c + 1 < cb.size(); c++) wmax = std::max(wmax, cb[c + 1] - cb[c]);
        for (int b = 0; b < 2; b++) P3_TRY(grow(&ctx->chunk_in[b], &ctx->chunk_in_bytes[b], h * wmax * 4, ctx->stream));
        P3_CUDA(cudaEventRecord(ctx->ev_start, ctx->stream));
        P3_CUDA(cudaStreamWaitEvent(ctx->h2d_stream, ctx->ev_start, 0));
        for (size_t c = 0; c + 1 < cb.size(); c++) {
            const int b = (int)(c & 1);
            const size_t c0 = cb[c], wc = cb[c + 1] - c0;
            if (c >= 2) P3_CUDA(cudaStreamWaitEvent(ctx->h2d_stream, ctx->ev_comp[b], 0));
            P3_CUDA(cudaMemcpy2DAsync(ctx->chunk_in[b], wc * 4, h_evals + c0, w * 4, wc * 4, h, cudaMemcpyHostToDevice, ctx->h2d_stream));
            P3_CUDA(cudaEventRecord(ctx->ev_h2d[b], ctx->h2d_stream));
            P3_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_h2d[b], 0));
            P3_TRY(ntt_coset_lde(ctx, field, (const u32 *)ctx->chunk_in[b], h, wc, log_blowup, shift, d_lde + c0, 1, wc, w));
            P3_CUDA(cudaEventRecord(ctx->ev_comp[b], ctx->stream));
        }
    }
    const u32 *mats[1] = {d_lde};
    const size_t lh = h << log_blowup;
    P3_TRY(hash_merkle_commit(ctx, field, hash, 1, mats, &lh, &w, d_layers, layer_lens, n_layers));
    const size_t nl = *n_layers, eff = cap_height < nl - 1 ? cap_height : nl - 1;
    size_t off = 0;
    for (size_t k = 0; k + 1 + eff < nl; k++) off += layer_lens[k];
    *cap_len = std::min((size_t)1 << eff, layer_lens[nl - 1 - eff]);
    P3_CUDA(cudaMemcpyAsync(h_cap, d_layers + off * 8, *cap_len * 32, cudaMemcpyDeviceToHost, ctx->stream));
    P3_CUDA(cudaStreamSynchronize(ctx->stream));
    return P3GPU_OK;
}

}  // extern "C"
