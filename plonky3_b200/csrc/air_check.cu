// The debug constraint check of any AIR given as a constraint program (air_program.cuh): p3_air::check_constraints /
// check_all_constraints (air/src/check_constraints.rs:429-627) on the device, over the trace domain.
//
// Mapping: one thread per trace row, a persistent grid sweeping the rows.  The instruction stream is the quotient kernel's (read with
// uniform loads, so opcodes never diverge), interpreted by air_row_check with the reference's debug semantics; a FOLD tests its slot
// for zero instead of accumulating an alpha power.  Slots live in a global-memory scratch laid out [slot][thread] over the whole
// grid, so a warp's slot accesses are 128 contiguous bytes; a check program may have up to 65,535 slots (SHA-256's has 6,711), far
// beyond what shared memory holds.  The grid is sized so that the scratch stays under AIR_CHECK_SCRATCH_BYTES, but at least one
// block per SM (DESIGN.md section 4.14).
//
// Two passes keep the report deterministic: pass 1 writes every row's failure count; pass 2 walks a given list of rows, one thread
// per row, and writes each row's failing constraint indices in ascending order at the row's given offset.
#include "common.h"
#include "air_program.cuh"

namespace p3 {

constexpr size_t AIR_CHECK_SCRATCH_BYTES = size_t(1) << 30;
constexpr unsigned AIR_CHECK_BLOCKS_PER_SM = 16;      // 2048 resident threads per SM at 128 threads per block

struct AirCheckArgs {
    const AirInsn *prog;
    u32 n_insns;
    const u32 *trace;
    size_t width;
    u32 height;
    const u32 *pre;             // preprocessed trace, height x pre_width (null without preprocessed columns)
    size_t pre_width;
    const u32 *periodic;        // periodic_rows x n_periodic, row-major (null without periodic columns)
    u32 n_periodic, periodic_rows;
    const u32 *pubs;
    u32 *scratch;               // slot s of grid thread t at scratch[s * threads + t]
    size_t threads;
    u32 *counts;                // pass 1: height failure counts
    const u32 *rows;            // pass 2: n_rows rows, their first output index and the output
    const u64 *offsets;
    u32 n_rows;
    u32 *failed;
};

template <int F> struct AirCheckEnv {
    const AirCheckArgs *a;
    u32 *sl;
    const u32 *row, *nrow, *prow, *pnrow, *per;
    __device__ __forceinline__ AirInsn insn(u32 pc) const {
        const uint2 v = __ldg(reinterpret_cast<const uint2 *>(a->prog) + pc);
        return AirInsn{v.x, v.y};
    }
    __device__ __forceinline__ u32 &slot(u32 s) { return sl[s * a->threads]; }
    __device__ __forceinline__ void set_rows(u32 i, u32 in) { row = a->trace + (size_t)i * a->width; nrow = a->trace + (size_t)in * a->width; }
    __device__ __forceinline__ void set_ext_rows(u32 i, u32 in, u32 pr) {
        prow = a->pre + (size_t)i * a->pre_width; pnrow = a->pre + (size_t)in * a->pre_width; per = a->periodic + (size_t)pr * a->n_periodic;
    }
    __device__ __forceinline__ u32 local(u32 c) const { return __ldg(row + c); }
    __device__ __forceinline__ u32 next(u32 c) const { return __ldg(nrow + c); }
    __device__ __forceinline__ u32 pre_local(u32 c) const { return __ldg(prow + c); }
    __device__ __forceinline__ u32 pre_next(u32 c) const { return __ldg(pnrow + c); }
    __device__ __forceinline__ u32 periodic(u32 k) const { return __ldg(per + k); }
    __device__ __forceinline__ u32 pub(u32 k) const { return __ldg(a->pubs + k); }
};

template <int F, bool LIST> __global__ void __launch_bounds__(AIR_BLOCK) air_check_kernel(const AirCheckArgs a) {
    const size_t t = (size_t)blockIdx.x * AIR_BLOCK + threadIdx.x;
    AirCheckEnv<F> env;
    env.a = &a;
    env.sl = a.scratch + t;
    const size_t n = LIST ? a.n_rows : a.height;
    for (size_t j = t; j < n; j += a.threads) {
        if constexpr (LIST) {
            u32 *out = a.failed + a.offsets[j];
            auto put = [&](u32 k) { *out++ = k; };
            air_row_check<F>(env, a.n_insns, a.rows[j], a.height, a.periodic_rows, put);
        } else {
            u32 c = 0;
            auto count = [&](u32) { c++; };
            air_row_check<F>(env, a.n_insns, (u32)j, a.height, a.periodic_rows, count);
            a.counts[j] = c;
        }
    }
}

// pass 1 (d_counts != null) or pass 2 (the row list); every argument is checked before anything launches
int32_t air_check(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *d_trace, size_t height, const u32 *d_pre, const u32 *d_periodic,
                  size_t periodic_rows, const u32 *pubs, u32 *d_counts, const u32 *d_rows, size_t n_rows, const u64 *d_offsets, u32 *d_failed) {
    P3_CHECK(pg->device == ctx->device, P3GPU_EINVAL, "AIR program was created on device %d, the context is on device %d", pg->device, ctx->device);
    P3_CHECK(pg->check, P3GPU_EINVAL, "the AIR program was not created with p3gpu_air_check_program_create");
    const AirProgram &p = pg->prog;
    const int field = p.field;
    const u32 P = field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    P3_CHECK(height >= 1 && height <= (1u << 31), P3GPU_EINVAL, "trace height %zu: need 1 <= height <= 2^31", height);
    P3_CHECK(reinterpret_cast<uintptr_t>(d_trace) % 4 == 0, P3GPU_EINVAL, "check: misaligned trace");
    P3_CHECK(p.n_public == 0 || pubs != nullptr, P3GPU_EINVAL, "the program reads %u public values, none given", p.n_public);
    for (u32 k = 0; k < p.n_public; k++) P3_CHECK(pubs[k] < P, P3GPU_EINVAL, "public value %u is not a canonical Montgomery word", k);
    P3_CHECK((p.pre_width > 0) == (d_pre != nullptr), P3GPU_EINVAL, "preprocessed trace %s, the program's preprocessed width is %u",
             d_pre ? "given" : "missing", p.pre_width);
    P3_CHECK(reinterpret_cast<uintptr_t>(d_pre) % 4 == 0, P3GPU_EINVAL, "check: misaligned preprocessed trace");
    P3_CHECK((p.n_periodic > 0) == (d_periodic != nullptr), P3GPU_EINVAL, "periodic table %s, the program has %u periodic columns",
             d_periodic ? "given" : "missing", p.n_periodic);
    if (d_periodic) {
        P3_CHECK(periodic_rows >= 1 && periodic_rows <= (1u << 31), P3GPU_EINVAL, "periodic table of %zu rows: need 1 <= rows <= 2^31", periodic_rows);
        P3_CHECK(reinterpret_cast<uintptr_t>(d_periodic) % 4 == 0, P3GPU_EINVAL, "check: misaligned periodic table");
    } else {
        periodic_rows = 0;
    }
    const bool list = d_counts == nullptr;
    if (list) {
        P3_CHECK(n_rows < (1u << 31), P3GPU_EINVAL, "%zu rows listed: at most 2^31 - 1", n_rows);
        if (n_rows == 0) return P3GPU_OK;
        P3_CHECK(reinterpret_cast<uintptr_t>(d_rows) % 4 == 0 && reinterpret_cast<uintptr_t>(d_offsets) % 8 == 0 &&
                     reinterpret_cast<uintptr_t>(d_failed) % 4 == 0, P3GPU_EINVAL, "check: misaligned row list, offsets or output");
        std::vector<u32> rows(n_rows);
        P3_CUDA(cudaMemcpyAsync(rows.data(), d_rows, n_rows * 4, cudaMemcpyDeviceToHost, ctx->stream));
        P3_CUDA(cudaStreamSynchronize(ctx->stream));
        for (size_t j = 0; j < n_rows; j++) P3_CHECK(rows[j] < height, P3GPU_EINVAL, "listed row %zu is %u, the trace has %zu rows", j, rows[j], height);
    } else {
        P3_CHECK(reinterpret_cast<uintptr_t>(d_counts) % 4 == 0, P3GPU_EINVAL, "check: misaligned counts");
    }

    AirCheckArgs ca;
    ca.prog = pg->d_insns; ca.n_insns = (u32)p.insns.size();
    ca.trace = d_trace; ca.width = p.width; ca.height = (u32)height;
    ca.pre = d_pre; ca.pre_width = p.pre_width;
    ca.periodic = d_periodic; ca.n_periodic = p.n_periodic; ca.periodic_rows = (u32)periodic_rows;
    ca.counts = d_counts; ca.rows = d_rows; ca.offsets = d_offsets; ca.n_rows = (u32)n_rows; ca.failed = d_failed;
    ca.pubs = nullptr;
    if (p.n_public) {
        void *tab = nullptr;
        P3_TRY(ctx_scratch2(ctx, (size_t)p.n_public * 4, &tab));
        P3_CUDA(cudaMemcpyAsync(tab, pubs, (size_t)p.n_public * 4, cudaMemcpyHostToDevice, ctx->stream));
        ca.pubs = static_cast<const u32 *>(tab);
    }
    // persistent grid: n_slots x threads x 4 B of scratch <= AIR_CHECK_SCRATCH_BYTES, but at least one block per SM
    const size_t work = list ? n_rows : height, block_bytes = (size_t)std::max<u32>(p.n_slots, 1) * AIR_BLOCK * 4;
    size_t blocks = std::max<size_t>(ctx->sm_count, AIR_CHECK_SCRATCH_BYTES / block_bytes);
    blocks = std::min(std::min(blocks, (size_t)ctx->sm_count * AIR_CHECK_BLOCKS_PER_SM), (work + AIR_BLOCK - 1) / AIR_BLOCK);
    ca.threads = blocks * AIR_BLOCK;
    void *scratch = nullptr;
    P3_CUDA(cudaMallocAsync(&scratch, blocks * block_bytes, ctx->stream));
    ca.scratch = static_cast<u32 *>(scratch);
    auto kern = field == BABY_BEAR ? (list ? air_check_kernel<BABY_BEAR, true> : air_check_kernel<BABY_BEAR, false>)
                                   : (list ? air_check_kernel<KOALA_BEAR, true> : air_check_kernel<KOALA_BEAR, false>);
    kern<<<(unsigned)blocks, AIR_BLOCK, 0, ctx->stream>>>(ca);
    ctx->launches++;
    const cudaError_t launched = cudaGetLastError();
    P3_CUDA(cudaFreeAsync(scratch, ctx->stream));
    P3_CUDA(launched);
    return P3GPU_OK;
}

}  // namespace p3
