// Batched NTT / coset LDE for row-major matrices over BabyBear / KoalaBear on sm_90a.
//
// Replaces Radix2DitParallel (dft/src/radix_2_dit_parallel.rs:30-515) behind TwoAdicSubgroupDft
// (dft/src/traits.rs:28-291).  Not a port: the reference runs two cache-blocked half networks separated by
// row bit-reversals on CPU threads; here ONE kernel family implements a Cooley-Tukey network that maps
// natural-order input to bit-reversed-order output ("network order"), executed as 1-3 passes over HBM:
//
//   * a pass owns the butterfly layers [l0, l1) of the size-2^n network.  A CTA takes a tile of R = 2^(l1-l0)
//     rows (all rows that agree on the top l0 and the low n-l1 index bits) x CT adjacent columns, stages it in
//     shared memory, runs the layers as radix-16 register steps (4 layers per shared-memory round trip), and
//     writes the tile back.  Row segments of CT*4 bytes are contiguous, so any row permutation (bit reversal on
//     input or output) is free: it only changes which 64/128-byte segments a tile touches.
//   * layer l uses one twiddle per block q (the reference's "twiddles with the coset shift baked in",
//     radix_2_dit_parallel.rs:80-115):  z_l[q] = shift^(N/2^(l+1)) * w_(2^(l+1))^bitrev_l(q).  They live in a
//     heap-ordered table Z[2^l + q]; a tile needs R-1 of them (contiguous runs per layer) and stages them in
//     shared memory next to the data.
//   * butterflies use Shoup multiplication by the precomputed twiddle and lazy [0, 2p) reduction:
//     3 multiply-pipe + 6 ALU-pipe instructions each (field.cuh: ct_butterfly).
//
// Two kernel generations implement a pass: ntt_pass_pipe_kernel (TMA tile loads into an mbarrier stage ring, warp-specialised
// consumer groups, column-tile-major intermediates) and ntt_pass_fast_kernel / ntt_pass_kernel (cp.async or plain loads).
// On H100 the cp.async kernel is the faster one for dense passes of 10 layers (2^20 rows: two such passes), the TMA pipeline
// for shorter passes (see pipe_mode).  The pipeline also runs the LDEs only it can do: a column block of a wider matrix
// (row pitch != width) and the row-sharded multi-GPU LDE.  P3GPU_NTT_PIPE=1 / 0 puts every eligible pass on it / none.
//
// coset_lde_batch = inverse network (root^-1, scale 1/h) producing coefficients in network (bit-reversed) order,
// then per coset a forward network reading those coefficients through a bit-reversed row map and leaving the
// evaluations in network order — which is exactly the bit-reversed row order the reference leaves in memory
// (radix_2_dit_parallel.rs:245, fri/src/two_adic_pcs.rs:313-318).  No standalone bit-reversal or scaling pass exists.
// With two equal passes on the cp.async kernel (2^20 rows by default) the LDE is three launches: inverse pass 1, ONE fused
// pass (ntt_lde_mid_kernel: inverse pass 2 and every coset's forward pass 1, tile by tile through shared memory and registers)
// and forward pass 2, so the coefficients are written and read once.  Forward pass 2 runs on whole-row bands in 8-CTA clusters
// (ntt_band_pass_kernel: one bulk copy per eighth of a band in and out, the three cross-CTA layers over distributed shared
// memory, overlapped with another band's local layers) where an eighth fits its ring slot; matrices of up to 48 columns keep
// 4-CTA clusters without the overlap (ntt_band_pass_narrow_kernel).  On the 8-CTA kernel with whole column tiles, the fused pass
// stores each tile from registers as one dense block of a tile-major scratch and forward pass 2 gathers its rows from those blocks
// (make_tile_major_tensor_maps): the corner turn between the two passes is done by tensor loads, not by short strided stores.
// Inverse pass 1 runs on the same kernel where a part fits
// (100 columns at 2^20 rows, 100-200 at 2^18), its "bands" being the strided units of rows 2^10 apart, each part moved by one 3-D
// tensor copy.
// Every other LDE runs the four passes as separate launches.
// The fused pass runs warp-specialised where its registers allow (all instances but the runtime-width one at r = 10): a producer
// lane loads each tile with one tensor copy and, on the dense plan, owns the tile stores and their read-out waits (DESIGN 4.1).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda.h>   // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint, no libcuda link)

#include "common.h"

namespace p3 {

// Phase-breakdown instrumentation (tools/ntt_timeline.py) is compiled in only with -DP3GPU_NTT_PROFILE; the env switches
// P3GPU_NTT_NOBFLY / NOLOAD / NOSTORE are ignored by the production build.
#ifdef P3GPU_NTT_PROFILE
#define P3_SKIP(flag) (flag)
#else
#define P3_SKIP(flag) false
#endif

static int env_int(const char *name, int dflt) {
    const char *s = getenv(name);
    return s ? atoi(s) : dflt;
}

// Profiling build: each launch gets its own 1 MiB window of the timeline buffer (8 windows, reused in turn).
static unsigned long long *prof_window() {
#ifdef P3GPU_NTT_PROFILE
    static int launch_no = 0;
    const char *pb = getenv("P3GPU_NTT_PROFBUF");
    return pb ? reinterpret_cast<unsigned long long *>(strtoull(pb, nullptr, 0)) + (size_t)(launch_no++ % 8) * (1u << 17) : nullptr;
#else
    return nullptr;
#endif
}

struct PassArgs {
    const u32 *in;
    u32 *out;
    u32 w;         // row pitch in elements
    u32 col0;      // first column of this launch
    u32 n_ctiles;  // column tiles (of CT columns) in this launch
    u32 ct;        // tile width of the generic-width kernel variant
    u32 n_cosets;  // cosets batched in this launch (fastest-varying part of blockIdx.x)
    u32 vec16;     // fast kernel: row segments are 16-byte aligned (cp.async 16)
    u32 tma_store; // fast kernel (inverse pass 1 of the three-launch LDE): step 2 writes the tile back to shared memory and ONE tensor copy stores it
    u32 skip_load, skip_store;  // profiling experiments only
    u32 skip_bfly; // profiling experiment only (P3GPU_NTT_NOBFLY=1): move the data, skip the butterflies
    u32 wc;                    // pipelined kernel: columns of this launch (<= w = row pitch of the dense layout)
    u32 in_tiled, out_tiled;   // pipelined kernel: intermediate buffers in column-tile-major layout (see lde_tiled_impl)
    u32 in_blocks;             // pipelined kernel, tiled input: 2^log_n-row blocks per column tile (cosets)
    u32 n_items, csplit, tpi;  // pipelined kernel: work items = (row tile, coset) units x csplit column chunks of tpi tiles
    unsigned long long *prof;  // profiling build only: per CTA/tile phase timestamps (P3GPU_NTT_PROFBUF)
    int log_n, l0, l1;
    const uint2 *tw;  // heap-ordered twiddles of coset 0
    int in_bitrev, out_bitrev;
    int out_sh;
    u32 out_add;  // output row = (maybe_bitrev(i) << out_sh) + out_add
    uint2 scale;
    int has_scale, final_reduce;
    size_t tw_stride;   // uint2 elements between consecutive cosets' heaps
    size_t out_stride;  // u32 elements between consecutive cosets' output blocks
    size_t in_stride;   // u32 elements between consecutive cosets' input blocks
    // Row-sharded output over peer memory (multi-GPU commit, last pass of the LDE only; pipelined kernel, dense output):
    // LDE row (coset << log_n) + i belongs to rank row >> shard_log_rows and is stored at that rank's buffer
    // shard_out[rank] (already offset to this launch's first column), local row = row & (2^shard_log_rows - 1), pitch w.
    // The buffers are this GPU's own block plus the peers' blocks mapped through CUDA IPC: the all-to-all that re-shards
    // column blocks into row blocks happens in the pass's own stores, tile by tile, over NVLink.
    u32 *shard_out[16];
    int shard_log_rows;   // 0 = off
};

template <int LOG_CT> __device__ __forceinline__ u32 sidx(u32 row, u32 c) {
    // XOR swizzle so that narrow column tiles (CT < 32) stay bank-conflict free in the stride-1 radix step
    if (LOG_CT < 5) row ^= (row >> 4) & ((32u >> LOG_CT) - 1u);
    return (row << LOG_CT) + c;
}

template <int F, int LOG_CT, int THREADS, int Q>
__device__ __forceinline__ void radix_step(u32 *data, const uint2 *tws, int r, int lam0) {
    constexpr u32 CT = 1u << LOG_CT;
    constexpr int E = 1 << Q;
    const int logD = r - lam0 - Q;
    const u32 D = 1u << logD;
    const u32 items = (1u << (r - Q)) << LOG_CT;
    for (u32 it = threadIdx.x; it < items; it += THREADS) {
        const u32 c = it & (CT - 1), g = it >> LOG_CT;
        const u32 lo = g & (D - 1), hi = g >> logD;
        const u32 base = (hi << (logD + Q)) + lo;
        const u32 node = (1u << lam0) + hi;
        u32 x[E];
#pragma unroll
        for (int m = 0; m < E; m++) x[m] = data[sidx<LOG_CT>(base + m * D, c)];
#pragma unroll
        for (int j = 0; j < Q; j++) {
            const int half = E >> (j + 1);
#pragma unroll
            for (int grp = 0; grp < (1 << j); grp++) {
                const uint2 z = tws[(node << j) + grp];
#pragma unroll
                for (int t = 0; t < half; t++) ct_butterfly<F>(x[grp * 2 * half + t], x[grp * 2 * half + t + half], z);
            }
        }
#pragma unroll
        for (int m = 0; m < E; m++) data[sidx<LOG_CT>(base + m * D, c)] = x[m];
    }
    __syncthreads();
}

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async8(void *smem, const void *gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(smem)), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// The twiddles of a tile of 2^r rows of the pass over layers [l0, l0 + r), row tile T (the top l0 row bits): layer l0 + lam uses the
// 2^lam contiguous heap entries from Z[2^(l0+lam) + T*2^lam], staged in shared memory as tws[2^lam + q] = Z[2^(l0+lam) + T*2^lam + q],
// so that tws is the heap of the tile's own r-layer network (tws[0] unused).  Every thread of the CTA copies entries
// threadIdx.x + 1, + THREADS, ... < 2^r; ASYNC: as cp.async copies in the caller's current group.  (load_tile_twiddles: the same
// table as bulk copies.)  l0 is taken by reference so that a kernel parameter passed there is read where it is used, as a
// constant-bank operand, not held in a register across the copy loop (whose asm statements keep the compiler from hoisting it).
template <int THREADS, bool ASYNC>
__device__ __forceinline__ void stage_tile_twiddles(uint2 *tws, const uint2 *tw, const int &l0, u32 T, u32 R) {
    for (u32 k = threadIdx.x + 1; k < R; k += THREADS) {
        const int lam = 31 - __clz(k);
        const uint2 *src = tw + ((size_t)1 << (l0 + lam)) + ((size_t)T << lam) + (k - (1u << lam));
        if constexpr (ASYNC) cp_async8(tws + k, src);
        else tws[k] = *src;
    }
}

template <int F, int LOG_CT, int THREADS, bool VEC>
__global__ void __launch_bounds__(THREADS) ntt_pass_kernel(const PassArgs a) {
    constexpr u32 CT = 1u << LOG_CT;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int r = a.l1 - a.l0;
    const u32 R = 1u << r;
    u32 *data = reinterpret_cast<u32 *>(smem_raw);
    uint2 *tws = reinterpret_cast<uint2 *>(data + ((size_t)R << LOG_CT));

    const u32 coset = blockIdx.x % a.n_cosets, bx = blockIdx.x / a.n_cosets;
    const u32 ctile = bx % a.n_ctiles, tile = bx / a.n_ctiles;
    const int lowbits = a.log_n - a.l1;
    const u32 L = tile & ((1u << lowbits) - 1u), T = tile >> lowbits;
    const u32 col = a.col0 + ctile * CT;
    const uint2 *tw = a.tw + (size_t)coset * a.tw_stride;
    const u32 *in = a.in + (size_t)coset * a.in_stride;
    u32 *out = a.out + (size_t)coset * a.out_stride;
    const u32 out_add = a.out_add;
    const u32 ibase = (a.l0 == 0 ? 0u : (T << (a.log_n - a.l0))) | L;
    const int brsh = 32 - a.log_n;

    stage_tile_twiddles<THREADS, false>(tws, tw, a.l0, T, R);
    // gather the tile
    if (VEC) {
        constexpr u32 CV = CT >= 4 ? CT / 4 : 1;
        for (u32 it = threadIdx.x; it < R * CV; it += THREADS) {
            const u32 c4 = it % CV, rho = it / CV;
            const u32 i = ibase | (rho << lowbits);
            const u32 row = a.in_bitrev ? (__brev(i) >> brsh) : i;
            uint4 v = *reinterpret_cast<const uint4 *>(in + (size_t)row * a.w + col + 4 * c4);
            if (a.has_scale) {
                v.x = shoup_mul<F>(v.x, a.scale); v.y = shoup_mul<F>(v.y, a.scale);
                v.z = shoup_mul<F>(v.z, a.scale); v.w = shoup_mul<F>(v.w, a.scale);
            }
            *reinterpret_cast<uint4 *>(data + sidx<LOG_CT>(rho, 4 * c4)) = v;
        }
    } else {
        for (u32 it = threadIdx.x; it < (R << LOG_CT); it += THREADS) {
            const u32 c = it & (CT - 1), rho = it >> LOG_CT;
            const u32 i = ibase | (rho << lowbits);
            const u32 row = a.in_bitrev ? (__brev(i) >> brsh) : i;
            u32 v = in[(size_t)row * a.w + col + c];
            if (a.has_scale) v = shoup_mul<F>(v, a.scale);
            data[sidx<LOG_CT>(rho, c)] = v;
        }
    }
    __syncthreads();

    int lam0 = 0;
    const int q0 = (r & 3) ? (r & 3) : 4;
    switch (q0) {
        case 1: radix_step<F, LOG_CT, THREADS, 1>(data, tws, r, 0); break;
        case 2: radix_step<F, LOG_CT, THREADS, 2>(data, tws, r, 0); break;
        case 3: radix_step<F, LOG_CT, THREADS, 3>(data, tws, r, 0); break;
        default: radix_step<F, LOG_CT, THREADS, 4>(data, tws, r, 0); break;
    }
    for (lam0 = q0; lam0 < r; lam0 += 4) radix_step<F, LOG_CT, THREADS, 4>(data, tws, r, lam0);

    // scatter the tile
    if (VEC) {
        constexpr u32 CV = CT >= 4 ? CT / 4 : 1;
        for (u32 it = threadIdx.x; it < R * CV; it += THREADS) {
            const u32 c4 = it % CV, rho = it / CV;
            const u32 i = ibase | (rho << lowbits);
            const u32 row = ((a.out_bitrev ? (__brev(i) >> brsh) : i) << a.out_sh) + out_add;
            uint4 v = *reinterpret_cast<const uint4 *>(data + sidx<LOG_CT>(rho, 4 * c4));
            if (a.final_reduce) { v.x = fp_reduce<F>(v.x); v.y = fp_reduce<F>(v.y); v.z = fp_reduce<F>(v.z); v.w = fp_reduce<F>(v.w); }
            *reinterpret_cast<uint4 *>(out + (size_t)row * a.w + col + 4 * c4) = v;
        }
    } else {
        for (u32 it = threadIdx.x; it < (R << LOG_CT); it += THREADS) {
            const u32 c = it & (CT - 1), rho = it >> LOG_CT;
            const u32 i = ibase | (rho << lowbits);
            const u32 row = ((a.out_bitrev ? (__brev(i) >> brsh) : i) << a.out_sh) + out_add;
            u32 v = data[sidx<LOG_CT>(rho, c)];
            if (a.final_reduce) v = fp_reduce<F>(v);
            out[(size_t)row * a.w + col + c] = v;
        }
    }
}

// ---- fast path: the whole pass as TWO register networks with one shared-memory exchange ------------------------
// For 7 <= r <= 10 the r layers split as Q1 + Q2 (Q2 = ceil(r/2) <= 5).  Step 1 loads 2^Q1 rows per thread straight from
// global memory (stride 2^Q2 local rows), runs Q1 layers in registers and parks the results in shared memory; step 2
// reads 2^Q2 consecutive local rows, runs Q2 layers and stores straight to global memory.  Per element and pass that is
// one shared store + one shared load (the generic kernel does 2 per radix step plus the staging copy).
// Shared layout: local row rho, column c at (rho >> Q2) * gstride + (rho & (2^Q2-1)) * CT + c with gstride = 2^Q2*CT + pad,
// pad chosen so that gstride = CT (mod 32): both access patterns are bank-conflict free for ANY tile width CT, which lets
// one launch class take a non-power-of-two remainder tile (e.g. 100 = 5 x 16 + 20 columns) without sector over-fetch.
template <int Q> __host__ __device__ constexpr u32 brev_const(u32 m) {
    u32 r = 0;
    for (int b = 0; b < Q; b++) r |= ((m >> b) & 1u) << (Q - 1 - b);
    return r;
}

// One layer per template instance: every loop bound is a compile-time constant, so the loops unroll fully and x stays in
// registers.  (As one loop nest, the inner bound E >> (j + 1) is constant only once the layer loop is unrolled; the sm_90a
// compiler unrolls in the other order, leaves a runtime loop and moves x to local memory: more than twice the LDE time.)
template <int F, int Q, int J>
__device__ __forceinline__ void reg_layer(u32 (&x)[1 << Q], const uint2 *tws, u32 node) {
    constexpr int half = (1 << Q) >> (J + 1);
#pragma unroll
    for (int grp = 0; grp < (1 << J); grp++) {
        const uint2 z = tws[(node << J) + grp];
#pragma unroll
        for (int t = 0; t < half; t++) ct_butterfly<F>(x[grp * 2 * half + t], x[grp * 2 * half + t + half], z);
    }
    if constexpr (J + 1 < Q) reg_layer<F, Q, J + 1>(x, tws, node);
}
template <int F, int Q>
__device__ __forceinline__ void reg_network(u32 (&x)[1 << Q], const uint2 *tws, u32 node) {
    reg_layer<F, Q, 0>(x, tws, node);
}

// Tile stores through the tensor copy engine: the tile's writers make their shared-memory writes visible to the async proxy,
// meet at a barrier, and one thread stores the whole tile with ONE 5-D tensor copy (box = the padded tile layout: see
// make_pass_tensor_map).  The copy drains to HBM while the SM computes; a buffer is rewritten only after
// bulk_wait_read says the copy has read it out of shared memory.
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_tile(const CUtensorMap *map, const void *smem, int c0, int c3, int c4) {
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                 ::"l"(reinterpret_cast<unsigned long long>(map)), "r"((u32)__cvta_generic_to_shared(smem)), "r"(c0), "r"(0), "r"(0), "r"(c3), "r"(c4)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// The same store with an L2 evict-last hint: the fused LDE pass writes each output row as short segments from several tiles,
// which should merge in L2 before they go to HBM, and the next pass reads them back.
__device__ __forceinline__ void tma_store_tile_keep(const CUtensorMap *map, const void *smem, int c0, int c3, int c4) {
    unsigned long long policy;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(policy));
    asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3, %4, %5, %6}], [%1], %7;"
                 ::"l"(reinterpret_cast<unsigned long long>(map)), "r"((u32)__cvta_generic_to_shared(smem)), "r"(c0), "r"(0), "r"(0), "r"(c3), "r"(c4), "l"(policy)
                 : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// mbarriers and bulk loads (the producer-warp form of ntt_lde_mid_kernel, and ntt_pass_pipe_kernel)
__device__ __forceinline__ void mbar_init(u32 bar, u32 count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_wait(u32 bar, u32 parity) {
    u32 done = 0, spins = 0;
    unsigned long long t0 = 0;
    while (true) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (done) break;
        // watchdog: a pass takes milliseconds; a wait of 20 s can only be a protocol error.  Trap (the launch fails with an error the
        // host reports) instead of leaving a hung kernel on the device.
        if ((++spins & 0xfffu) == 0) {
            unsigned long long now;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            if (t0 == 0) t0 = now;
            else if (now - t0 > 20000000000ull) __trap();
        }
    }
}
// The same wait without a watchdog, for a barrier that only a thread whose own waits have one arrives on (it then cannot hang
// unless that thread traps): no registers beyond its operands, for waits at a kernel's register cap.
__device__ __forceinline__ void mbar_wait_plain(u32 bar, u32 parity) {
    asm volatile("{ .reg .pred p; WAIT_%=: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1; @!p bra WAIT_%=; }" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(u32 bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_arrive_n(u32 bar, u32 n) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(u32 bar, u32 bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_load(void *smem, const void *gmem, u32 bytes, u32 bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"((u32)__cvta_generic_to_shared(smem)), "l"(gmem), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_tile(const CUtensorMap *map, void *smem, int c0, int c3, int c4, u32 bar) {
    asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
                 ::"r"((u32)__cvta_generic_to_shared(smem)), "l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(0), "r"(0), "r"(c3), "r"(c4),
                   "r"(bar) : "memory");
}
// a tile's twiddle table of stage_tile_twiddles, layers 1 <= lam < r: one bulk copy per layer on `bar`, 8 * (2^r - 2) bytes.
// Layer 0's single 8-byte entry tws[1] = Z[2^l0 + T] is too small for a bulk copy: the producer writes it itself, before its
// arrive on bar.
__device__ __forceinline__ void load_tile_twiddles(uint2 *tws, const uint2 *tw, int l0, u32 T, int r, u32 bar) {
#pragma unroll 1
    for (int lam = 1; lam < r; lam++) bulk_load(tws + (1u << lam), tw + ((size_t)1 << (l0 + lam)) + ((size_t)T << lam), 8u << lam, bar);
}
// Consumer-only barrier of a producer-warp kernel (the producer warp never joins it); the plain kernels use __syncthreads.
template <bool PROD, u32 THREADS> __device__ __forceinline__ void consumer_sync() {
    if constexpr (PROD) asm volatile("bar.sync 1, %0;" ::"n"(THREADS) : "memory");
    else __syncthreads();
}

// Persistent, double-buffered pass kernel.  A CTA (one per SM) walks over tiles of 2^R_LOG rows x `ct` columns:
//   * tile k+1 (rows as 16-byte cp.async/LDGSTS copies, plus its 2^R_LOG - 1 twiddles) streams into the second shared
//     buffer while tile k is computed, so HBM latency overlaps the integer work;
//   * step 1 runs Q1 layers in registers IN PLACE in shared memory, step 2 runs Q2 layers and either streams the results to
//     global memory from registers or (a.tma_store: inverse pass 1 of the three-launch LDE) writes them back in place and
//     the tile leaves as ONE tensor copy that drains while the next tile computes.  (One 1-D bulk copy per row segment was
//     rejected: UBLKCP is a warp-uniform instruction, so one copy per lane serialises into a 32-iteration loop per warp.)
//   * all tiles of a pass have the same runtime width ct (16/20/24 columns; w = 100 -> 5 x 20) so that ONE launch covers
//     every column and neighbouring tiles share DRAM bursts through L2.
template <int F, int R_LOG, int CT_T, int THREADS, int NBUF>   // CT_T: compile-time tile width (16/20/24) or 0 = runtime a.ct
__global__ void __launch_bounds__(THREADS, NBUF == 2 ? 1 : (CT_T == 16 && THREADS == 256) ? 3 : 2)
ntt_pass_fast_kernel(const __grid_constant__ PassArgs a, const __grid_constant__ CUtensorMap omap) {
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    constexpr u32 E1 = 1u << Q1, E2 = 1u << Q2, R = 1u << R_LOG;
    const u32 CT = CT_T ? (u32)CT_T : a.ct;
    const u32 padw = (CT + 32u - ((E2 * CT) & 31u)) & 31u;
    const u32 gstride = E2 * CT + padw;
    const u32 buf_words = (E1 * gstride + 3u) & ~3u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u32 *data0 = reinterpret_cast<u32 *>(smem_raw);
    uint2 *tws0 = reinterpret_cast<uint2 *>(data0 + NBUF * buf_words);

    const int lowbits = a.log_n - a.l1;
    const int brsh = 32 - a.log_n;
    const u32 n_row_tiles = 1u << (a.log_n - R_LOG);
    const u32 total = n_row_tiles * a.n_ctiles * a.n_cosets;
    const bool vec16 = a.vec16 != 0;       // row segments 16-byte aligned in global memory (loads AND stores)
    const bool shared_tw = (a.l0 == 0);    // first pass of a network: every tile uses the same twiddles
    const bool tma_store = NBUF == 2 && a.tma_store;   // the output map omap is set up (launch_fast_rct)

    auto decode = [&](u32 t, u32 &coset, u32 &col, u32 &cw, u32 &T, u32 &ibase) {
        coset = t % a.n_cosets;
        const u32 bx = t / a.n_cosets;
        const u32 ctile = bx % a.n_ctiles, tile = bx / a.n_ctiles;
        const u32 L = tile & ((1u << lowbits) - 1u);
        T = tile >> lowbits;
        col = ctile * CT;
        cw = min(CT, a.w - col);
        ibase = (a.l0 == 0 ? 0u : (T << (a.log_n - a.l0))) | L;
    };
    auto issue = [&](u32 t, u32 buf) {
        u32 coset, col, cw, T, ibase;
        decode(t, coset, col, cw, T, ibase);
        u32 *data = data0 + buf * buf_words;
        const u32 *in = a.in + (size_t)coset * a.in_stride + col;
        if (!shared_tw || a.n_cosets > 1) stage_tile_twiddles<THREADS, true>(tws0 + buf * R, a.tw + (size_t)coset * a.tw_stride, a.l0, T, R);
        // chunk = 16 bytes (4 columns) when aligned, else one element
        const u32 cpr = vec16 ? (cw >> 2) : cw;                  // chunks per row segment
        const u32 rs = (THREADS / cpr) & ~(E2 - 1u);             // rows per sweep: a multiple of E2 keeps the shared address linear
        const u32 nthr = rs * cpr;
        if (rs == 0) {
            // fewer than E2 whole rows per sweep (wide unaligned tiles): plain index arithmetic per chunk
            for (u32 it = threadIdx.x; it < R * cpr; it += THREADS) {
                const u32 rho = it / cpr, ch = it - rho * cpr;
                const u32 e = vec16 ? 4u * ch : ch;
                const u32 i = ibase | (rho << lowbits);
                const u32 row = a.in_bitrev ? (__brev(i) >> brsh) : i;
                u32 *dst = data + (rho >> Q2) * gstride + (rho & (E2 - 1u)) * CT + e;
                const u32 *src = in + (size_t)row * a.w + e;
                if (vec16) cp_async16(dst, src); else cp_async4(dst, src);
            }
        } else if (threadIdx.x < nthr) {
            const u32 rho0 = threadIdx.x / cpr, ch = threadIdx.x - rho0 * cpr;
            const u32 e = vec16 ? 4u * ch : ch;
            u32 *dst = data + (rho0 >> Q2) * gstride + (rho0 & (E2 - 1u)) * CT + e;
            const u32 dstep = (rs >> Q2) * gstride;
            if (!a.in_bitrev) {
                const u32 *src = in + (size_t)(ibase | (rho0 << lowbits)) * a.w + e;
                const size_t sstep = ((size_t)rs << lowbits) * a.w;
                for (u32 rho = rho0; rho < R; rho += rs, dst += dstep, src += sstep) {
                    if (vec16) cp_async16(dst, src); else cp_async4(dst, src);
                }
            } else {
                for (u32 rho = rho0; rho < R; rho += rs, dst += dstep) {
                    const u32 row = __brev(ibase | (rho << lowbits)) >> brsh;
                    const u32 *src = in + (size_t)row * a.w + e;
                    if (vec16) cp_async16(dst, src); else cp_async4(dst, src);
                }
            }
        }
        cp_async_commit();
    };

    u32 t = blockIdx.x;
    if (t >= total) return;
#ifdef P3GPU_NTT_PROFILE
    // 8 slots per (CTA, tile < 16): smid, t_start, t_issued, t_loaded, t_step1, t_step2 (globaltimer ns)
#define P3_STAMP(slot) do { if (a.prof && threadIdx.x == 0 && k < 16) { unsigned long long ts_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts_)); \
        a.prof[((size_t)blockIdx.x * 16 + k) * 8 + (slot)] = ts_; } } while (0)
#else
#define P3_STAMP(slot) do { } while (0)
#endif
    if (shared_tw && a.n_cosets == 1) stage_tile_twiddles<THREADS, true>(tws0, a.tw, a.l0, 0, R);   // once per CTA, lands with the first tile's group
    if (NBUF == 2) issue(t, 0);
    for (u32 k = 0; t < total; t += gridDim.x, k++) {
        const u32 buf = NBUF == 2 ? (k & 1u) : 0u;
        if (tma_store && threadIdx.x == 0) bulk_wait_read();   // the previous tile's store has left the buffer refilled next
        __syncthreads();   // every warp is done reading the buffer that is refilled next
#ifdef P3GPU_NTT_PROFILE
        if (a.prof && threadIdx.x == 0 && k < 16) { u32 sm_; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm_)); a.prof[((size_t)blockIdx.x * 16 + k) * 8] = sm_; }
#endif
        P3_STAMP(1);
        if (NBUF == 2) {
            if (t + gridDim.x < total) { issue(t + gridDim.x, buf ^ 1u); cp_async_wait<1>(); }
            else cp_async_wait<0>();
        } else {   // single buffer: other resident CTAs of this SM compute while this one waits for its tile
            if (!P3_SKIP(a.skip_load)) issue(t, 0);
            P3_STAMP(2);
            cp_async_wait<0>();
        }
        __syncthreads();
        P3_STAMP(3);
        u32 *data = data0 + buf * buf_words;
        const uint2 *tws = (shared_tw && a.n_cosets == 1) ? tws0 : tws0 + buf * R;  // NBUF == 1: buf == 0
        u32 coset, col, cw, T, ibase;
        decode(t, coset, col, cw, T, ibase);
        const u32 dg = THREADS / cw, dc = THREADS - dg * cw;
        // ---- step 1 (in place in shared memory): item (g, c) holds local rows g + m*E2, m < E1
        {
            u32 g = threadIdx.x / cw, c = threadIdx.x - g * cw;
            for (; g < E2; ) {
                u32 *sp = data + g * CT + c;
                u32 x[E1];
#pragma unroll
                for (u32 m = 0; m < E1; m++) x[m] = sp[m * gstride];
                if (a.has_scale) {
#pragma unroll
                    for (u32 m = 0; m < E1; m++) x[m] = shoup_mul<F>(x[m], a.scale);
                }
                if (!P3_SKIP(a.skip_bfly)) reg_network<F, Q1>(x, tws, 1u);
#pragma unroll
                for (u32 m = 0; m < E1; m++) sp[m * gstride] = x[m];
                c += dc; g += dg;
                if (c >= cw) { c -= cw; g++; }
            }
        }
        __syncthreads();
        P3_STAMP(4);
        // ---- step 2: item (g, c) holds local rows g*E2 + m, m < E2
        {
            u32 *out = a.out + (size_t)coset * a.out_stride + col;
            // out row(m) = ((row0 + K_m * S) << out_sh) + out_add: natural: K_m = m, S = 1 << lowbits;
            //                                                        bit-reversed: K_m = brev_Q2(m), S = 1 << (l0+Q1)
            const size_t sstride = ((size_t)(a.out_bitrev ? (1u << (a.l0 + Q1)) : (1u << lowbits)) << a.out_sh) * a.w;
            u32 g = threadIdx.x / cw, c = threadIdx.x - g * cw;
            for (; g < E1; ) {
                u32 *sp = data + g * gstride + c;
                u32 x[E2];
#pragma unroll
                for (u32 m = 0; m < E2; m++) x[m] = sp[m * CT];
                if (!P3_SKIP(a.skip_bfly)) reg_network<F, Q2>(x, tws, E1 + g);
                if (a.final_reduce) {
#pragma unroll
                    for (u32 m = 0; m < E2; m++) x[m] = fp_reduce<F>(x[m]);
                }
                if (tma_store) {
                    if (!P3_SKIP(a.skip_store)) {
#pragma unroll
                        for (u32 m = 0; m < E2; m++) sp[m * CT] = x[m];
                    }
                } else {
                    const u32 i0 = ibase | (g << (lowbits + Q2));
                    const u32 row0 = ((a.out_bitrev ? (__brev(i0) >> brsh) : i0) << a.out_sh) + a.out_add;
                    u32 *p = out + (size_t)row0 * a.w + c;
                    if (P3_SKIP(a.skip_store)) { u32 acc = 0;
#pragma unroll
                        for (u32 m = 0; m < E2; m++) acc ^= x[m];
                        if (acc == 0x12345678u) p[0] = acc;
                    } else if (a.out_bitrev) {
#pragma unroll
                        for (u32 m = 0; m < E2; m++) p[brev_const<Q2>(m) * sstride] = x[m];
                    } else {
#pragma unroll
                        for (u32 m = 0; m < E2; m++) p[m * sstride] = x[m];
                    }
                }
                c += dc; g += dg;
                if (c >= cw) { c -= cw; g++; }
            }
            if (tma_store && !P3_SKIP(a.skip_store)) {
                fence_proxy_async_smem();
                __syncthreads();
                // tensor coordinates (column, 0, 0, L, T + coset block): see make_pass_tensor_map
                if (threadIdx.x == 0) tma_store_tile(&omap, data, (int)col, (int)(ibase & ((1u << lowbits) - 1u)), (int)(T + (coset << a.l0)));
            }
        }
        P3_STAMP(5);
    }
    if (tma_store && threadIdx.x == 0) bulk_wait_all();
}

// ---- last pass of the two-pass coset LDE on whole-row bands, in clusters of CL CTAs ------------------------------------
// The forward networks' second pass (layers [n - R, n)) of coset block `coset` works on bands of 2^R CONTIGUOUS rows: band T is
// rows T*2^R .. (T+1)*2^R - 1, one contiguous run of 2^R * w words in memory.  A cluster of CL CTAs takes a band, CTA q its rows
// [q*RQ, (q+1)*RQ), RQ = 2^R / CL (its "part"): the part comes in as ONE 1-D bulk copy and leaves as ONE, with no row segments,
// partial sectors or per-thread addresses.
//   * step X: the band's first log2(CL) layers pair rows 2^R/2 .. RQ apart, i.e. row j of every part: one radix-CL step over
//     distributed shared memory, CTA q taking rows j in [q*RQ/CL, (q+1)*RQ/CL) of the CL parts (ld/st.shared::cluster);
//   * steps A and B: the remaining layers pair rows inside a part: two register steps on the part in place (as steps 1 and
//     2 of ntt_pass_fast_kernel), then the final reduction;
//   * three warp roles run at once, each on its own band, in "periods" that end with ONE cluster barrier of every thread: in
//     period k the exchange warps run step X on band k+1, the local warps steps A and B on band k (exchanged in period k-1), and
//     the copy warp keeps a 3-slot ring (band k in slot k % 3).  The barrier at the end of period k certifies that every peer has
//     finished exchanging band k+1, that every CTA holds band k+2 (the copy warp waits its `full` mbarrier before arriving), and
//     that nobody still reads a peer's slot the next period reuses;
//   * the copy lane stores band k as soon as the local warps are done with it (named barrier 2), arrives on the cluster barrier,
//     and only then waits until that store has read slot k % 3 out and loads band k+3 there (the thread that commits a bulk group
//     is the one that can wait for it), so the read-out and the load overlap the next period's work.  Band k+3 is waited on at
//     the end of period k+1.
// Threads are laid along columns (item = row * w + column): every warp access to shared memory is a run of consecutive words.
constexpr int BAND_XWARPS = 6, BAND_LWARPS = 14;   // exchange and local warps (chosen by measurement, DESIGN 4.1), plus the copy warp
constexpr int BAND_THREADS = 32 * (BAND_XWARPS + BAND_LWARPS + 1), BAND_NARROW_THREADS = 512;
constexpr size_t BAND_SLOT_BYTES = 50 * 1024;   // the largest part a ring slot takes (2^R/CL rows x w x 4 bytes)

__device__ __forceinline__ u32 cluster_rank() { u32 r; asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned; barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ u32 cluster_map(u32 smem_addr, u32 rank) {
    u32 r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ uint4 ld_cluster_v4(u32 addr) {
    uint4 v;
    asm volatile("ld.shared::cluster.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void st_cluster_v4(u32 addr, uint4 v) {
    asm volatile("st.shared::cluster.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void bulk_store(void *gmem, const void *smem, u32 bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem), "r"((u32)__cvta_generic_to_shared(smem)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// a strided unit's part through a 3-D tensor map (column, unit, row of the unit): see make_unit_tensor_map
__device__ __forceinline__ void tma_load_part(const CUtensorMap *map, void *smem, u32 unit, u32 row0, u32 bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"((u32)__cvta_generic_to_shared(smem)), "l"(reinterpret_cast<unsigned long long>(map)), "r"(0), "r"(unit), "r"(row0), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void tma_store_part(const CUtensorMap *map, const void *smem, u32 unit, u32 row0) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(reinterpret_cast<unsigned long long>(map)), "r"((u32)__cvta_generic_to_shared(smem)), "r"(0), "r"(unit), "r"(row0) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// Block row of forward row i = j * 2^Q1 + b (j < 2^Q2, b < 2^Q1: forward step 2's item j, register b, with Q1 and Q2 as
// ntt_lde_mid_kernel splits r) in a tile-major block: b * 2^Q2 + j, so that register b of consecutive items is one contiguous run.
// The map moves bit fields, so it splits over them: tile_block_row(j * 2^Q1 + b) = tile_block_row(j * 2^Q1) + tile_block_row(b).
template <int R_LOG> __host__ __device__ constexpr u32 tile_block_row(u32 i) {
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    return ((i & ((1u << Q1) - 1u)) << Q2) + (i >> Q1);
}
// its inverse: the forward row i that block row p holds
template <int R_LOG> __host__ __device__ constexpr u32 tile_block_row_inv(u32 p) {
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    return ((p & ((1u << Q2) - 1u)) << Q1) + (p >> Q2);
}
static_assert(tile_block_row_inv<7>(tile_block_row<7>(37)) == 37 && tile_block_row<7>(37) == 5 * 16 + 4, "tile-major block rows");
// a band's part gathered from the tile-major scratch through a 5-D tensor map (column, column tile, block row, tile row, coset): see
// make_tile_major_tensor_maps
__device__ __forceinline__ void tma_load_gather(const CUtensorMap *map, void *smem, u32 T, u32 l0, u32 coset, u32 bar) {
    asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
                 ::"r"((u32)__cvta_generic_to_shared(smem)), "l"(reinterpret_cast<unsigned long long>(map)), "r"(0), "r"(0), "r"(T), "r"(l0),
                   "r"(coset), "r"(bar) : "memory");
}

// The band's layers as both band kernels split them: LX cross-CTA layers (step X), then QA (step A) and QB (step B) local layers
// on each CTA's part of RQ rows.
template <int R_LOG, int CL> struct BandShape {
    static constexpr int LX = CL == 8 ? 3 : CL == 4 ? 2 : 1;
    static constexpr int QB = (R_LOG - LX + 1) / 2, QA = R_LOG - LX - QB;
    static constexpr u32 RQ = 1u << (R_LOG - LX), R = 1u << R_LOG;
    static_assert(CL == 1 << LX && QA >= 1, "band pass: cluster size");
};

// The steps of one band on the CTA's part `part` (w columns) with the band's twiddles `tws`, run by THREADS threads of which the
// caller is thread t.  A kernel's profiling build skips them with P3GPU_NTT_NOBFLY (bit 1: step X, bit 0: steps A and B).
// ---- step X: rows j + p*RQ, p < CL, j in CTA q's share; x[p] lives in CTA p.  An item is 4 adjacent columns: one 16-byte access
// per peer needs a quarter of the instructions of word accesses and keeps 4x the bytes in flight (the exchange is bound by the
// latency of remote shared memory, not by its bandwidth).
template <int F, int R_LOG, int CL, u32 THREADS>
__device__ __forceinline__ void band_step_x(const PassArgs &a, u32 *part, const uint2 *tws, u32 w, u32 q, u32 t) {
    using S = BandShape<R_LOG, CL>;
    u32 peer[CL];
#pragma unroll
    for (int p = 0; p < CL; p++) peer[p] = cluster_map((u32)__cvta_generic_to_shared(part), (u32)p);
    const u32 items = P3_SKIP(a.skip_bfly & 2) ? 0 : (S::RQ / CL) * (w / 4), base = 16 * q * items;
    for (u32 it = t; it < items; it += THREADS) {
        const u32 off = base + 16 * it;
        uint4 v[CL];
#pragma unroll
        for (int p = 0; p < CL; p++) v[p] = ld_cluster_v4(peer[p] + off);
#pragma unroll
        for (int e = 0; e < 4; e++) {
            u32 x[CL];
#pragma unroll
            for (int p = 0; p < CL; p++) x[p] = (&v[p].x)[e];
            reg_network<F, S::LX>(x, tws, 1u);
#pragma unroll
            for (int p = 0; p < CL; p++) (&v[p].x)[e] = x[p];
        }
#pragma unroll
        for (int p = 0; p < CL; p++) st_cluster_v4(peer[p] + off, v[p]);
    }
}
// ---- step A: item (g, c) holds local rows g + m * 2^QB, m < 2^QA (layers LX .. LX+QA-1 of block q)
template <int F, int R_LOG, int CL, u32 THREADS>
__device__ __forceinline__ void band_step_a(const PassArgs &a, u32 *part, const uint2 *tws, u32 w, u32 q, u32 t) {
    using S = BandShape<R_LOG, CL>;
    for (u32 it = t; it < (P3_SKIP(a.skip_bfly & 1) ? 0 : w << S::QB); it += THREADS) {
        u32 *sp = part + it;
        u32 x[1 << S::QA];
#pragma unroll
        for (u32 m = 0; m < (1u << S::QA); m++) x[m] = sp[m * (w << S::QB)];
        reg_network<F, S::QA>(x, tws, (1u << S::LX) + q);
#pragma unroll
        for (u32 m = 0; m < (1u << S::QA); m++) sp[m * (w << S::QB)] = x[m];
    }
}
// ---- step B: item (g, c) holds local rows g * 2^QB + m, m < 2^QB; then the scale by a.scale (SCALE and a.has_scale) and the
// final reduction (a.final_reduce)
template <int F, int R_LOG, int CL, u32 THREADS, bool SCALE>
__device__ __forceinline__ void band_step_b(const PassArgs &a, u32 *part, const uint2 *tws, u32 w, u32 q, u32 t) {
    using S = BandShape<R_LOG, CL>;
    for (u32 it = t; it < (P3_SKIP(a.skip_bfly & 1) ? 0 : w << S::QA); it += THREADS) {
        const u32 g = it / w, c = it - g * w;
        u32 *sp = part + (g << S::QB) * w + c;
        u32 x[1 << S::QB];
#pragma unroll
        for (u32 m = 0; m < (1u << S::QB); m++) x[m] = sp[m * w];
        reg_network<F, S::QB>(x, tws, (1u << (S::LX + S::QA)) + (q << S::QA) + g);
        if (SCALE && a.has_scale) {
#pragma unroll
            for (u32 m = 0; m < (1u << S::QB); m++) x[m] = shoup_mul<F>(x[m], a.scale);
        }
        if (a.final_reduce) {
#pragma unroll
            for (u32 m = 0; m < (1u << S::QB); m++) x[m] = fp_reduce<F>(x[m]);
        }
#pragma unroll
        for (u32 m = 0; m < (1u << S::QB); m++) sp[m * w] = x[m];
    }
}
// A contiguous band's part (not STRIDED): CTA q's RQ rows of band T of coset block `coset` come in as ONE bulk copy into `part`,
// the band's twiddles as load_tile_twiddles' copies into `tws`, both on mbarrier `bar`; they leave as ONE bulk copy.
template <int R_LOG, int CL>
__device__ __forceinline__ void band_load_part(const PassArgs &a, u32 *part, uint2 *tws, u32 coset, u32 T, u32 q, u32 bar) {
    using S = BandShape<R_LOG, CL>;
    const uint2 *tw = a.tw + (size_t)coset * a.tw_stride;
    const u32 qwords = S::RQ * a.w;
    tws[1] = tw[((size_t)1 << a.l0) + T];
    const bool load = !P3_SKIP(a.skip_load);
    mbar_expect_tx(bar, (load ? qwords * 4 : 0) + 8 * (S::R - 2));
    if (load) bulk_load(part, a.in + (size_t)coset * a.in_stride + ((size_t)T * S::R + q * S::RQ) * a.w, qwords * 4, bar);
    load_tile_twiddles(tws, tw, a.l0, T, R_LOG, bar);
}
template <int R_LOG, int CL>
__device__ __forceinline__ void band_store_part(const PassArgs &a, const u32 *part, u32 coset, u32 T, u32 q) {
    using S = BandShape<R_LOG, CL>;
    bulk_store(a.out + (size_t)coset * a.out_stride + ((size_t)T * S::R + q * S::RQ) * a.w, part, S::RQ * a.w * 4);
}

// a: l0 = log_n - R_LOG, l1 = log_n (rows of a band contiguous), dense in / out blocks of a.n_cosets cosets, w % 4 == 0, 16-byte aligned.
// STRIDED: the first pass of a network instead (l0 = 0, l1 = R_LOG, one block, no pitch).  Its "band" T is the strided unit of rows
// T + 2^(log_n - R_LOG) * i, i < 2^R_LOG, so the same network runs on the unit's index i.  CTA q's part, rows i in [q*RQ, (q+1)*RQ),
// comes in as ONE 3-D tensor copy (imap) and leaves as ONE 3-D tensor store (omap); every unit uses the same twiddles Z[1..2^R),
// loaded once with slot 0's first load.  The network is linear, so the scale by a.scale is applied where the values leave step B, on
// the 14 local warps: in step X it made the 6 exchange warps the ones that set the period (DESIGN 4.1).  The ring has a fourth slot,
// which the one twiddle table leaves room for.
// GATHER: the last pass of the LDE reading the fused pass's tile-major scratch a.in (launch_lde_mid) instead of a dense block: CTA q's
// part of band T, rows L in [q*RQ, (q+1)*RQ), is block row tile_block_row(T) of the blocks of tiles L, and comes in as ONE 5-D tensor copy (imap,
// make_tile_major_tensor_maps) whose box lands as the same row-major part.  A cluster's bands go in block-row order (out_of).
// Everything else is the contiguous band's.
template <int F, int R_LOG, int CL, bool GATHER, bool STRIDED>
__global__ void __launch_bounds__(BAND_THREADS, 1)
ntt_band_pass_kernel(const __grid_constant__ PassArgs a, const __grid_constant__ CUtensorMap imap, const __grid_constant__ CUtensorMap omap) {
    static_assert(!(GATHER && STRIDED), "the gather mode is the last pass's");
    constexpr u32 RQ = BandShape<R_LOG, CL>::RQ, R = 1u << R_LOG;
    constexpr u32 NX = 32 * BAND_XWARPS, NL = 32 * BAND_LWARPS;    // threads [0, NX) exchange, [NX, NX + NL) local, then the copy warp
    constexpr u32 NS = STRIDED ? 4 : 3;                            // ring slots
    constexpr u32 TW_SLOTS = STRIDED ? 1 : NS;                     // twiddle tables: one per ring slot, or the one all units share
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const u32 w = a.w;
    const u32 qwords = RQ * w;                                     // one part
    u32 *data0 = reinterpret_cast<u32 *>(smem_raw);
    uint2 *tws0 = reinterpret_cast<uint2 *>(data0 + NS * qwords);
    unsigned long long *full = reinterpret_cast<unsigned long long *>(tws0 + TW_SLOTS * R);
    const u32 full_a = (u32)__cvta_generic_to_shared(full);
    const u32 q = cluster_rank();
    const u32 n_clusters = gridDim.x / CL, cid = blockIdx.x / CL;
    const int band_log = a.log_n - R_LOG;
    const u32 total = a.n_cosets << band_log;
    const int n = (int)((total - 1 - cid) / n_clusters) + 1;      // this cluster's bands: cid + k * n_clusters, k < n (grid <= bands)

    // GATHER: the bands in block-row order, so that the clusters at work at once gather neighbouring block rows, which share lines
    auto out_of = [&](u32 k, u32 &coset, u32 &T) {
        const u32 t = cid + k * n_clusters;
        coset = t >> band_log;
        T = t & ((1u << band_log) - 1u);
        if constexpr (GATHER) T = tile_block_row_inv<R_LOG>(T);
    };
    auto issue = [&](u32 k) {   // copy lane: band k's part and twiddles into ring slot k % NS
        u32 coset, T;
        out_of(k, coset, T);
        const u32 s = k % NS;
        const u32 bar = full_a + 8 * s;
        if constexpr (STRIDED) {
            const bool load = !P3_SKIP(a.skip_load), tw = k == 0;
            if (tw) tws0[1] = a.tw[1];
            mbar_expect_tx(bar, (load ? qwords * 4 : 0) + (tw ? 8 * (R - 2) : 0));
            if (load) tma_load_part(&imap, data0 + s * qwords, T, q * RQ, bar);
            if (tw) load_tile_twiddles(tws0, a.tw, 0, 0, R_LOG, bar);
        } else if constexpr (GATHER) {
            const uint2 *tw = a.tw + (size_t)coset * a.tw_stride;
            uint2 *tws = tws0 + s * R;
            const bool load = !P3_SKIP(a.skip_load);
            tws[1] = tw[((size_t)1 << a.l0) + T];
            mbar_expect_tx(bar, (load ? qwords * 4 : 0) + 8 * (R - 2));
            if (load) tma_load_gather(&imap, data0 + s * qwords, tile_block_row<R_LOG>(T), q * RQ, coset, bar);
            load_tile_twiddles(tws, tw, a.l0, T, R_LOG, bar);
        } else {
            band_load_part<R_LOG, CL>(a, data0 + s * qwords, tws0 + s * R, coset, T, q, bar);
        }
    };
    auto wait_full = [&](u32 k) { mbar_wait(full_a + 8 * (k % NS), (k / NS) & 1u); };   // band k is slot k % NS's (k / NS)-th load

    const bool copy_warp = threadIdx.x >= NX + NL, copy_lane = threadIdx.x == NX + NL;
    if (threadIdx.x == 0) {
        for (u32 s = 0; s < NS; s++) mbar_init(full_a + 8 * s, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (copy_lane)
        for (int k = 0; k < (int)NS && k < n; k++) issue(k);
    if (copy_warp) wait_full(0);
    cluster_sync_all();   // every CTA of the cluster holds its part of band 0
    // period k: exchange band k+1, local steps on band k; k = -1 only exchanges band 0
    for (int k = -1; k < n; k++) {
        if (threadIdx.x < NX) {
            if (k + 1 < n) {   // step X on band k+1
                const u32 s = (k + 1) % NS;
                band_step_x<F, R_LOG, CL, NX>(a, data0 + s * qwords, tws0 + (STRIDED ? 0 : s * R), w, q, threadIdx.x);
            }
            cluster_sync_all();
        } else if (!copy_warp) {
            if (k >= 0) {
                const u32 s = k % NS, lt = threadIdx.x - NX;
                u32 *data = data0 + s * qwords;
                const uint2 *tws = tws0 + (STRIDED ? 0 : s * R);
                band_step_a<F, R_LOG, CL, NL>(a, data, tws, w, q, lt);
                asm volatile("bar.sync 1, %0;" ::"n"(NL) : "memory");
                band_step_b<F, R_LOG, CL, NL, STRIDED>(a, data, tws, w, q, lt);
                fence_proxy_async_smem();
                asm volatile("bar.arrive 2, %0;" ::"n"(NL + 32) : "memory");   // band k may be stored
            }
            cluster_sync_all();
        } else {
            if (k + 2 < n) wait_full(k + 2);
            if (k >= 0) {
                asm volatile("bar.sync 2, %0;" ::"n"(NL + 32) : "memory");
                if (copy_lane && !P3_SKIP(a.skip_store)) {
                    u32 coset, T;
                    out_of(k, coset, T);
                    if constexpr (STRIDED) tma_store_part(&omap, data0 + (k % NS) * qwords, T, q * RQ);
                    else band_store_part<R_LOG, CL>(a, data0 + (k % NS) * qwords, coset, T, q);
                }
            }
            __syncwarp();
            cluster_arrive();
            if (copy_lane && k >= 0 && k + (int)NS < n) {
                bulk_wait_read();   // band k's store has read slot k % NS out
                issue(k + NS);
            }
            __syncwarp();
            cluster_wait();
        }
    }
    if (copy_lane) bulk_wait_all();
    cluster_sync_all();   // no CTA exits while a peer may still map its shared memory
}

// Narrow matrices: the same pass and steps in 4-CTA clusters with a 2-slot ring and no warp roles (every thread exchanges band k, then
// runs its steps A and B, while thread 0 loads band k+1).  With little work per band the pass is bound by its per-band barriers,
// and 4-CTA clusters (30 on the H100) take half as many bands each as 8-CTA clusters (15).
template <int F, int R_LOG, int CL>
__global__ void __launch_bounds__(BAND_NARROW_THREADS, 1) ntt_band_pass_narrow_kernel(const __grid_constant__ PassArgs a) {
    constexpr u32 NT = BAND_NARROW_THREADS, R = 1u << R_LOG;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const u32 w = a.w;
    const u32 qwords = BandShape<R_LOG, CL>::RQ * w;               // one quarter
    u32 *data0 = reinterpret_cast<u32 *>(smem_raw);
    uint2 *tws0 = reinterpret_cast<uint2 *>(data0 + 2 * qwords);
    unsigned long long *full = reinterpret_cast<unsigned long long *>(tws0 + 2 * R);
    const u32 full_a = (u32)__cvta_generic_to_shared(full);
    const u32 q = cluster_rank();
    const u32 n_clusters = gridDim.x / CL;
    const int band_log = a.log_n - R_LOG;
    const u32 total = a.n_cosets << band_log;

    auto issue = [&](u32 t, u32 buf) {   // thread 0: band t's quarter and twiddles into ring slot buf
        band_load_part<R_LOG, CL>(a, data0 + buf * qwords, tws0 + buf * R, t >> band_log, t & ((1u << band_log) - 1u), q, full_a + 8 * buf);
    };

    u32 t = blockIdx.x / CL;
    if (threadIdx.x == 0) {
        mbar_init(full_a, 1); mbar_init(full_a + 8, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        if (t < total) issue(t, 0);
    }
    __syncthreads();
    for (u32 k = 0; t < total; t += n_clusters, k++) {
        const u32 buf = k & 1u;
        u32 *data = data0 + buf * qwords;
        const uint2 *tws = tws0 + buf * R;
        mbar_wait(full_a + 8 * buf, (k >> 1) & 1u);
        cluster_sync_all();   // every CTA of the cluster holds its quarter of band t
        band_step_x<F, R_LOG, CL, NT>(a, data, tws, w, q, threadIdx.x);
        cluster_sync_all();   // every CTA has the exchanged values of its quarter; nobody touches a peer's buffer before the next band
        if (threadIdx.x == 0 && t + n_clusters < total) {
            bulk_wait_read();   // band k-1's store has read out the other buffer
            issue(t + n_clusters, buf ^ 1u);
        }
        band_step_a<F, R_LOG, CL, NT>(a, data, tws, w, q, threadIdx.x);
        __syncthreads();
        band_step_b<F, R_LOG, CL, NT, false>(a, data, tws, w, q, threadIdx.x);
        fence_proxy_async_smem();
        __syncthreads();
        if (threadIdx.x == 0 && !P3_SKIP(a.skip_store)) band_store_part<R_LOG, CL>(a, data, t >> band_log, t & ((1u << band_log) - 1u), q);
    }
    if (threadIdx.x == 0) bulk_wait_all();
}

// ---- fused middle passes of the two-pass coset LDE (2^(2r) rows, 7 <= r <= 10) ------------------------------------
// The inverse network's second pass (layers [r, 2r)) and the forward networks' first pass (layers [0, r), read through the
// bit-reversed row map) touch the same data tile by tile: inverse tile T holds coefficient rows T*2^r + rho, and forward tile
// L = bitrev_r(T) reads exactly those rows, its local row rho' = bitrev_r(rho).  One kernel does both, so the coefficients
// cross HBM once (read) instead of three times (write, re-read, scattered re-read):
//   * the tile (2^r contiguous rows x ct columns) and its inverse twiddles stream in with cp.async, double-buffered as in
//     ntt_pass_fast_kernel; the forward twiddles of every coset (layers [0, r): the same for every tile) are staged once;
//   * inverse step 1: Q1 layers in place in shared memory; inverse step 2: Q2 layers into registers.  A step-2 item holds local
//     rows g*E2 + m, i.e. forward rows bitrev_Q2(m)*E1 + bitrev_Q1(g): exactly one forward step-1 item (Q2 layers on rows
//     gf + j*E1, gf = bitrev_Q1(g)), so the coefficients stay in that thread's registers for all cosets;
//   * per coset: forward step 1 in registers, stored to the tile buffer in forward layout, then forward step 2 (Q1 layers) on
//     consecutive local rows, in place; ONE tensor copy (omap) stores the tile to that coset's output block, where the
//     four-launch path's forward pass 1 stores it; the next coset rewrites the buffer once the copy has read it out, and the HBM
//     writes drain while the CTA computes;
//   * TILES (the tile-major plan, make_tile_major_tensor_maps): forward step 2 stores its results from registers to the tile's
//     dense block of the scratch a.out instead, in the block-row order of tile_block_row, in which each warp's store of one
//     register is one whole 128-byte line.  No write-back, fence or read-out wait: the next coset's forward step 1 rewrites the
//     buffer once every warp's step 2 has read it (one consumer barrier);
//   * work items go in forward-tile order (L, column tile), T = bitrev_r(L): the CTAs resident at once store neighbouring
//     output rows (runs of ~26 rows per 2^r-row group at 132 SMs) instead of rows 2^r / 32 apart, while each tile's
//     reads stay one contiguous block of 2^r rows.
// THREADS = E1 * CT_T (E1 * 12 for the runtime-width variant) gives every forward step-1 item (E1*cw of them) its own thread.
// PROD (producer-warp form, every instance whose registers allow it: lde_mid_producer): one more warp, lane 0 of which loads the
// tile (ONE tensor copy, imap over the coefficients in the inverse layout; the zero-filled pad row per group is the shared layout)
// and its inverse twiddles (one bulk copy per layer) on full[b], stages the forward twiddles with the first tile, and owns the
// stores: the consumers write a coset's forward step 2 back, fence and arrive on ready[b]; the producer stores the tile, waits
// until the copy has read the buffer out (the thread that commits a bulk group is the one that can wait for it) and arrives on
// `freed`, which the consumers wait on before the next coset's forward step 1 rewrites the buffer.  After a tile's last coset
// the producer refills the buffer with tile k + 2 instead: the consumers' only other wait is full[b].  TILES: the producer stores
// nothing; the consumers arrive on ready[b] once per tile, after the last coset's step 2 has read the buffer, and the producer
// then refills it.
// (TILES precedes CT_T so that no instance's name ends in "true, false>", the band pass's gather instance: tests match on it.)
template <int R_LOG, int CT_T> __host__ __device__ constexpr int lde_mid_threads() { return (1 << (R_LOG / 2)) * (CT_T ? CT_T : 12); }

template <int F, int R_LOG, bool TILES, int CT_T, bool PROD>   // CT_T: compile-time tile width (16/20) or 0 = runtime a.ct (4/8/12)
__global__ void __launch_bounds__(lde_mid_threads<R_LOG, CT_T>() + (PROD ? 32 : 0), 1)
ntt_lde_mid_kernel(const __grid_constant__ PassArgs a, const uint2 *tw_fwd, const __grid_constant__ CUtensorMap omap,
                   const __grid_constant__ CUtensorMap imap) {
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    constexpr u32 E1 = 1u << Q1, E2 = 1u << Q2, R = 1u << R_LOG;
    constexpr u32 THREADS = lde_mid_threads<R_LOG, CT_T>();
    const u32 CT = CT_T ? (u32)CT_T : a.ct;
    const u32 gs1 = E2 * CT + ((CT + 32u - ((E2 * CT) & 31u)) & 31u);   // inverse layout: E1 groups of E2 local rows
    const u32 gs2 = E1 * CT + ((CT + 32u - ((E1 * CT) & 31u)) & 31u);   // forward layout: E2 groups of E1 local rows
    const u32 buf_words = (max(E1 * gs1, E2 * gs2) + 3u) & ~3u;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u32 *data0 = reinterpret_cast<u32 *>(smem_raw);
    uint2 *twi0 = reinterpret_cast<uint2 *>(data0 + 2 * buf_words);    // the tile's inverse twiddles, double-buffered
    uint2 *twf = twi0 + 2 * R;                                          // forward twiddles, R per coset
    // PROD: mbarriers full[b] (producer arrive + transaction bytes), ready[b] (every consumer thread, per coset), freed (producer)
    const u32 bar0 = (u32)__cvta_generic_to_shared(twf + a.n_cosets * R);
    auto full_bar = [&](u32 b) { return bar0 + 8u * b; };
    auto ready_bar = [&](u32 b) { return bar0 + 16u + 8u * b; };
    const u32 freed_bar = bar0 + 32u;

    const u32 total = (1u << (a.log_n - R_LOG)) * a.n_ctiles;
    auto issue = [&](u32 t, u32 buf) {
        const u32 ctile = t % a.n_ctiles, T = __brev(t / a.n_ctiles) >> (32 - R_LOG);
        const u32 col = ctile * CT, cw = min(CT, a.w - col);
        stage_tile_twiddles<THREADS, true>(twi0 + buf * R, a.tw, R_LOG, T, R);   // the inverse heap's layers [r, 2r)
        const u32 cpr = cw >> 2;                         // 16-byte chunks per row segment
        const u32 rs = (THREADS / cpr) & ~(E2 - 1u);     // rows per sweep, >= E2 because THREADS >= 4 * E1 * cpr
        if (threadIdx.x < rs * cpr) {
            const u32 rho0 = threadIdx.x / cpr, e = 4u * (threadIdx.x - rho0 * cpr);
            u32 *dst = data0 + buf * buf_words + (rho0 >> Q2) * gs1 + (rho0 & (E2 - 1u)) * CT + e;
            const u32 *src = a.in + ((size_t)T * R + rho0) * a.w + col + e;
            const u32 dstep = (rs >> Q2) * gs1;
            const size_t sstep = (size_t)rs * a.w;
            for (u32 rho = rho0; rho < R; rho += rs, dst += dstep, src += sstep) cp_async16(dst, src);
        }
        cp_async_commit();
    };

    u32 t = blockIdx.x;
    if (t >= total) return;
#ifdef P3GPU_NTT_PROFILE
    // PROD: the producer stamps slot 2 (load issue) and slot 6 (its wait for the tile's stores to be read out, summed over cosets)
#define P3_PSTAMP(kk, slot, v) do { if (a.prof && (kk) < 16) a.prof[((size_t)blockIdx.x * 16 + (kk)) * 8 + (slot)] = (v); } while (0)
#else
#define P3_PSTAMP(kk, slot, v) do { } while (0)
#endif
    if constexpr (PROD) {
        if (threadIdx.x == 0) {
            for (u32 b = 0; b < 2; b++) { mbar_init(full_bar(b), 1); mbar_init(ready_bar(b), THREADS); }
            if constexpr (!TILES) mbar_init(freed_bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (threadIdx.x >= THREADS) {
            // ---------------- producer ----------------
            if (threadIdx.x != THREADS) return;
            const u32 n_mine = (total - blockIdx.x + gridDim.x - 1) / gridDim.x;   // tiles of this CTA
            auto load = [&](u32 k) {
                const u32 b = k & 1u, tt = blockIdx.x + k * gridDim.x;
                const u32 col = (tt % a.n_ctiles) * CT, T = __brev(tt / a.n_ctiles) >> (32 - R_LOG);
                uint2 *tws = twi0 + b * R;
                tws[1] = a.tw[((size_t)1 << R_LOG) + T];
                // the box counts its zero-filled pad rows: E1 groups of gs1 = (E2 + 1) * CT words; the first tile brings the forward
                // twiddles of every coset (whole heaps of R entries: entry 0 is unused, but keeps the copy a multiple of 16 bytes)
                mbar_expect_tx(full_bar(b), E1 * gs1 * 4u + 8u * (R - 2u) + (k == 0 ? a.n_cosets * R * 8u : 0u));
#ifdef P3GPU_NTT_PROFILE
                { unsigned long long ts_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts_)); P3_PSTAMP(k, 2, ts_); }
#endif
                if (k == 0)
                    for (u32 cs = 0; cs < a.n_cosets; cs++) bulk_load(twf + cs * R, tw_fwd + (size_t)cs * a.tw_stride, R * 8u, full_bar(b));
                load_tile_twiddles(tws, a.tw, R_LOG, T, R_LOG, full_bar(b));
                // tensor coordinates (column, 0, 0, 0, T): coefficient rows T * 2^r + rho (see launch_lde_mid)
                tma_load_tile(&imap, data0 + b * buf_words, (int)col, 0, (int)T, full_bar(b));
            };
            load(0);
            if (n_mine > 1) load(1);
            for (u32 k = 0; k < n_mine; k++) {
                const u32 b = k & 1u, tt = blockIdx.x + k * gridDim.x;
                if constexpr (TILES) {
                    // ready[b] completes once per tile in buffer b, when its last coset's step 2 has read the buffer
                    mbar_wait(ready_bar(b), (k >> 1) & 1u);
                } else {
                    const u32 col = (tt % a.n_ctiles) * CT, L = tt / a.n_ctiles;
#ifdef P3GPU_NTT_PROFILE
                    unsigned long long read_wait = 0;
#endif
                    for (u32 cs = 0; cs < a.n_cosets; cs++) {
                        // ready[b] completes once per coset of every tile in buffer b
                        mbar_wait(ready_bar(b), ((k >> 1) * a.n_cosets + cs) & 1u);
                        if (!P3_SKIP(a.skip_store)) {
#ifdef P3GPU_NTT_PROFILE
                            unsigned long long w0_, w1_;
                            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(w0_));
#endif
                            // tensor coordinates (column, 0, 0, L, coset): see launch_lde_mid
                            tma_store_tile_keep(&omap, data0 + b * buf_words, (int)col, (int)L, (int)cs);
                            bulk_wait_read();   // the copy has read the buffer out: the next coset (or tile) may rewrite it
#ifdef P3GPU_NTT_PROFILE
                            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(w1_));
                            read_wait += w1_ - w0_;
#endif
                        }
                        if (cs + 1 < a.n_cosets) mbar_arrive(freed_bar);
                    }
#ifdef P3GPU_NTT_PROFILE
                    P3_PSTAMP(k, 6, read_wait);
#endif
                }
                if (k + 2 < n_mine) load(k + 2);
            }
            if constexpr (!TILES) bulk_wait_all();
            return;
        }
    } else {
        for (u32 k = threadIdx.x; k < a.n_cosets * R; k += THREADS)   // heap entries 1..R-1 of every coset (entry 0 is unused)
            if (k & (R - 1u)) cp_async8(twf + k, tw_fwd + (size_t)(k >> R_LOG) * a.tw_stride + (k & (R - 1u)));
        issue(t, 0);   // the forward twiddles land with the first tile's group
    }
    for (u32 k = 0; t < total; t += gridDim.x, k++) {
        const u32 buf = k & 1u;
        if constexpr (PROD) {
#ifdef P3GPU_NTT_PROFILE
            if (a.prof && threadIdx.x == 0 && k < 16) { u32 sm_; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm_)); a.prof[((size_t)blockIdx.x * 16 + k) * 8] = sm_; }
#endif
            P3_STAMP(1);
            mbar_wait(full_bar(buf), (k >> 1) & 1u);   // every consumer thread waits for every tile, in order
        } else {
            if (!TILES && threadIdx.x == 0) bulk_wait_read();   // the previous tile's last store has left the buffer refilled next
            __syncthreads();   // every warp is done with the buffer that is refilled next
#ifdef P3GPU_NTT_PROFILE
            if (a.prof && threadIdx.x == 0 && k < 16) { u32 sm_; asm volatile("mov.u32 %0, %%smid;" : "=r"(sm_)); a.prof[((size_t)blockIdx.x * 16 + k) * 8] = sm_; }
#endif
            P3_STAMP(1);
            if (t + gridDim.x < total) { issue(t + gridDim.x, buf ^ 1u); P3_STAMP(2); cp_async_wait<1>(); }
            else { P3_STAMP(2); cp_async_wait<0>(); }
            __syncthreads();
        }
        P3_STAMP(3);
        u32 *data = data0 + buf * buf_words;
        const uint2 *twi = twi0 + buf * R;
        const u32 ctile = t % a.n_ctiles, L = t / a.n_ctiles;
        const u32 col = ctile * CT, cw = min(CT, a.w - col);
        const u32 dg = THREADS / cw, dc = THREADS - dg * cw;
        // ---- inverse step 1 (in place): item (g, c) holds local rows g + m*E2
        {
            u32 g = threadIdx.x / cw, c = threadIdx.x - g * cw;
            for (; g < E2; ) {
                u32 *sp = data + g * CT + c;
                u32 x[E1];
#pragma unroll
                for (u32 m = 0; m < E1; m++) x[m] = sp[m * gs1];
                if (!P3_SKIP(a.skip_bfly)) reg_network<F, Q1>(x, twi, 1u);
#pragma unroll
                for (u32 m = 0; m < E1; m++) sp[m * gs1] = x[m];
                c += dc; g += dg;
                if (c >= cw) { c -= cw; g++; }
            }
        }
        consumer_sync<PROD, THREADS>();
        P3_STAMP(4);
        // ---- inverse step 2 into registers: thread (gf, c) takes inverse item g = bitrev_Q1(gf), local rows g*E2 + m.
        // (gf, not g, is linear in the thread index so that the per-coset stores below are bank-conflict free.)
        const u32 gf = threadIdx.x / cw, c = threadIdx.x - gf * cw;
        const bool active = gf < E1;
        u32 coef[E2];
        if (active) {
            const u32 g = __brev(gf) >> (32 - Q1);
            const u32 *sp = data + g * gs1 + c;
#pragma unroll
            for (u32 m = 0; m < E2; m++) coef[m] = sp[m * CT];
            if (!P3_SKIP(a.skip_bfly)) reg_network<F, Q2>(coef, twi, E1 + g);
        }
#ifdef P3GPU_NTT_PROFILE
        // slot 6 (PROD: 7): time thread 0 waits for the previous coset's store to leave the buffer (PROD: for the producer's `freed`;
        // TILES: for the barrier before forward step 1)
        unsigned long long store_wait = 0;
#endif
        for (u32 cs = 0; cs < a.n_cosets; cs++) {
            const uint2 *tf = twf + cs * R;
            // (Running forward step 1 before this wait keeps y[] live next to coef[] across it: 80 bytes of spills at r = 10, ct = 20.)
#ifdef P3GPU_NTT_PROFILE
            unsigned long long w0_ = 0, w1_ = 0;
            if (cs > 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(w0_));
#endif
            if constexpr (TILES) {
                consumer_sync<PROD, THREADS>();   // every warp's step 2 of the previous coset (cs = 0: inverse step 2) has read the buffer
            } else if (PROD && cs > 0) {
                // the producer has seen the previous coset's store leave the buffer: `freed` completes n_cosets - 1 times per tile.
                // coef[] is live here: at r = 10, ct = 20 a phase counter or the watchdog's registers would spill.
                mbar_wait_plain(freed_bar, (k * (a.n_cosets - 1u) + cs - 1u) & 1u);
            } else {
                if (cs > 0 && threadIdx.x == 0) bulk_wait_read();   // the previous coset's store has left the buffer
                consumer_sync<PROD, THREADS>();   // the tile buffer takes the forward layout (cs = 0: every warp is done with inverse step 2)
            }
#ifdef P3GPU_NTT_PROFILE
            if (cs > 0) { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(w1_)); store_wait += w1_ - w0_; }
#endif
            // ---- forward step 1: forward local rows gf + j*E1 = inverse local rows g*E2 + bitrev_Q2(j)
            if (active) {
                u32 y[E2];
#pragma unroll
                for (u32 j = 0; j < E2; j++) y[j] = coef[brev_const<Q2>(j)];
                if (!P3_SKIP(a.skip_bfly)) reg_network<F, Q2>(y, tf, 1u);
                u32 *sp = data + gf * CT + c;
#pragma unroll
                for (u32 j = 0; j < E2; j++) sp[j * gs2] = y[j];
            }
            consumer_sync<PROD, THREADS>();
            // ---- forward step 2 (in place; TILES: to the tile's block of coset cs, see make_tile_major_tensor_maps): item (j, c2)
            // holds forward local rows j*E1 + b, network rows L + (j*E1 + b) * 2^r
            if constexpr (TILES) {
                // cw = CT: item it = j*CT + c2 stores register b to block word tile_block_row(j*E1 + b)*CT + c2 = b*E2*CT + it, so a
                // warp's 32 consecutive items write one whole 128-byte line per register.  (32-bit word offsets: the scratch holds
                // fewer than 2^32 words, see coset_lde_impl.)
                const u32 blk = (cs * total + t) * R * CT;
                for (u32 it = threadIdx.x; it < E2 * CT; it += THREADS) {
                    const u32 j = it / CT, c2 = it - j * CT;
                    const u32 *sp = data + j * gs2 + c2;
                    u32 x[E1];
#pragma unroll
                    for (u32 b = 0; b < E1; b++) x[b] = sp[b * CT];
                    if (!P3_SKIP(a.skip_bfly)) reg_network<F, Q1>(x, tf, E2 + j);
                    if (!P3_SKIP(a.skip_store)) {
                        u32 *dst = a.out + blk + tile_block_row<R_LOG>(j * E1) * CT + c2;
#pragma unroll
                        for (u32 b = 0; b < E1; b++) dst[tile_block_row<R_LOG>(b) * CT] = x[b];
                    }
                }
            } else {
                u32 j = threadIdx.x / cw, c2 = threadIdx.x - j * cw;
                for (; j < E2; ) {
                    u32 *sp = data + j * gs2 + c2;
                    u32 x[E1];
#pragma unroll
                    for (u32 b = 0; b < E1; b++) x[b] = sp[b * CT];
                    if (!P3_SKIP(a.skip_bfly)) reg_network<F, Q1>(x, tf, E2 + j);
                    if (!P3_SKIP(a.skip_store)) {
#pragma unroll
                        for (u32 b = 0; b < E1; b++) sp[b * CT] = x[b];
                    }
                    c2 += dc; j += dg;
                    if (c2 >= cw) { c2 -= cw; j++; }
                }
            }
            if constexpr (TILES) {
                if (PROD && cs + 1 == a.n_cosets) {
                    // this thread's shared-memory writes are ordered before the producer's next load into this buffer; then the
                    // producer may refill it
                    fence_proxy_async_smem();
                    mbar_arrive(ready_bar(buf));
                }
            } else if constexpr (PROD) {
                // this thread's shared-memory writes are ordered before the producer's tensor copies (the store of this coset, and
                // after the last coset the next load into this buffer); then the producer may take the buffer
                fence_proxy_async_smem();
                mbar_arrive(ready_bar(buf));
            } else if (!P3_SKIP(a.skip_store)) {
                fence_proxy_async_smem();
                __syncthreads();
                // tensor coordinates (column, 0, 0, L, coset): see launch_lde_mid
                if (threadIdx.x == 0) tma_store_tile(&omap, data, (int)col, (int)L, (int)cs);
            }
        }
#ifdef P3GPU_NTT_PROFILE
        if (a.prof && threadIdx.x == 0 && k < 16) a.prof[((size_t)blockIdx.x * 16 + k) * 8 + (PROD ? 7 : 6)] = store_wait;
#endif
        P3_STAMP(5);
    }
    if (!PROD && !TILES && threadIdx.x == 0) bulk_wait_all();
}

// ---- pipelined path: TMA tile loads + warp-specialised consumer groups -------------------------------------------
// The cp.async kernel above spends a large share of each tile issuing and waiting for its own loads (LDGSTS issue is
// back-pressured by HBM latency, tools/ntt_timeline.py), and only 2-3 CTAs fit an SM.  This kernel
// keeps ONE CTA per SM and decouples the two jobs:
//   * a producer lane walks the CTA's tile sequence and issues ONE 5-D tiled TMA copy per tile (cp.async.bulk.tensor) into a
//     ring of NSTAGE shared-memory stages, plus the tile row's 2^r - 1 twiddles as 1-D bulk copies; completion is signalled
//     on mbarriers, so up to NSTAGE - NGROUP tiles (~34 KB each) are always in flight per SM at zero issue cost;
//   * NGROUP independent consumer groups (GTHREADS threads, own named barrier) each take every NGROUP-th tile through the same
//     two register networks as above and release the stage as soon as their last shared-memory read is done.
// Tiles are 2^r rows x 8 columns (32-byte row segments = one sector).  The TMA box is (8 cols, GS + 1, NG): asking for one
// row more than the tensor has in the "row within group" dimension makes the copy engine zero-fill a padding row per group,
// which is exactly the skew (group stride = 8 mod 32 words) that keeps both register-network access patterns bank-conflict
// free; no other padding mechanism exists for a dense TMA box.
// A CTA processes all column tiles of one (row tile, coset) unit back to back, so the unit's twiddles are staged once and
// neighbouring 32-byte segments of the same rows are requested within microseconds of each other (L2/DRAM page locality).
// PERM = the pass reads its rows through the bit-reversal map (first forward pass of the LDE): the tile is then a CONTIGUOUS
// block of rows holding local row rho at position bitrev_r(rho); the two steps simply swap their shared-memory access shapes.
template <int F, int R_LOG, bool PERM, int NSTAGE, int NGROUP, int GTHREADS>
__global__ void __launch_bounds__(NGROUP * GTHREADS + 32, 1) ntt_pass_pipe_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ PassArgs a) {
    constexpr u32 CT = 8;
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    constexpr u32 E1 = 1u << Q1, E2 = 1u << Q2, R = 1u << R_LOG;
    constexpr u32 GS = PERM ? E1 : E2, NG = PERM ? E2 : E1;   // rows per group, groups per tile (see above)
    constexpr u32 gstride = (GS + 1) * CT;
    constexpr u32 STAGE_WORDS = NG * gstride;
    constexpr u32 BOX_BYTES = STAGE_WORDS * 4;
    static_assert(BOX_BYTES % 128 == 0, "stage alignment");
    extern __shared__ __align__(128) unsigned char smem_raw[];
    u32 *stages = reinterpret_cast<u32 *>(smem_raw);
    uint2 *tws0 = reinterpret_cast<uint2 *>(smem_raw + (size_t)NSTAGE * BOX_BYTES);
    const u32 bar0 = (u32)__cvta_generic_to_shared(smem_raw + (size_t)NSTAGE * BOX_BYTES + 2 * R * sizeof(uint2));
    // barrier slots (8 bytes each): full[s] = s, empty[s] = NSTAGE + s, twfull[b] = 2 NSTAGE + b, twempty[b] = 2 NSTAGE + 2 + b
    auto full_bar = [&](u32 s) { return bar0 + 8u * s; };
    auto empty_bar = [&](u32 s) { return bar0 + 8u * (NSTAGE + s); };
    auto twfull_bar = [&](u32 b) { return bar0 + 8u * (2 * NSTAGE + b); };
    auto twempty_bar = [&](u32 b) { return bar0 + 8u * (2 * NSTAGE + 2 + b); };

    if (threadIdx.x == 0) {
        for (u32 s = 0; s < NSTAGE; s++) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), NGROUP * GTHREADS); }
        for (u32 b = 0; b < 2; b++) { mbar_init(twfull_bar(b), 1); mbar_init(twempty_bar(b), a.tpi * NGROUP * GTHREADS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int lowbits = a.log_n - a.l1;
    const int brsh = 32 - a.log_n;
    auto decode = [&](u32 it, u32 &coset, u32 &L, u32 &T, u32 &ct0, u32 &ct1) {
        const u32 unit = it / a.csplit, chunk = it - unit * a.csplit;
        coset = unit % a.n_cosets;
        const u32 tile = unit / a.n_cosets;
        L = tile & ((1u << lowbits) - 1u);
        T = tile >> lowbits;
        ct0 = chunk * a.tpi;
        ct1 = min(ct0 + a.tpi, a.n_ctiles);
    };

    if (threadIdx.x >= NGROUP * GTHREADS) {
        // ---------------- producer ----------------
        if ((threadIdx.x & 31u) != 0) return;
        u32 q = 0, ui = 0;
        for (u32 it = blockIdx.x; it < a.n_items; it += gridDim.x, ui++) {
            u32 coset, L, T, ct0, ct1;
            decode(it, coset, L, T, ct0, ct1);
            const u32 b = ui & 1u, ph = (ui >> 1) & 1u;
            mbar_wait(twempty_bar(b), ph ^ 1u);   // every tile of unit ui-2 is done with this twiddle buffer
            if (ct1 - ct0 < a.tpi) mbar_arrive_n(twempty_bar(b), (a.tpi - (ct1 - ct0)) * NGROUP * GTHREADS);   // short last chunk
            {
                const uint2 *tw = a.tw + (size_t)coset * a.tw_stride;
                uint2 *tws = tws0 + b * R;
                tws[1] = tw[((size_t)1 << a.l0) + T];
                mbar_expect_tx(twfull_bar(b), 8u * (R - 2u));
                load_tile_twiddles(tws, tw, a.l0, T, R_LOG, twfull_bar(b));
            }
            // tensor coordinates: (column, 0, 0, c3, c4); see make_pass_tensor_map
            // tiled input: column tile ct, block cb is the 8-column matrix number ct * in_blocks + cb (blocks fold into dim 4)
            const u32 in_block = (a.in_tiled ? a.in_blocks > 1 : a.in_stride != 0) ? coset : 0u;
            const int blk_sh = PERM ? lowbits : a.l0;   // dim-4 coordinates per 2^log_n-row block
            const int c3 = PERM ? 0 : (int)L;
            const int c4 = (PERM ? (lowbits ? (int)(__brev(L) >> (32 - lowbits)) : 0) : (int)T) + (int)(in_block << blk_sh);
            for (u32 ct = ct0; ct < ct1; ct++, q++) {
                const u32 s = q % NSTAGE, k = q / NSTAGE;
                mbar_wait(empty_bar(s), (k & 1u) ^ 1u);
                mbar_expect_tx(full_bar(s), BOX_BYTES);
                const int cc0 = a.in_tiled ? 0 : (int)(ct * CT);
                const int cc4 = a.in_tiled ? c4 + (int)((ct * a.in_blocks) << blk_sh) : c4;
                tma_load_tile(&tmap, stages + (size_t)s * STAGE_WORDS, cc0, c3, cc4, full_bar(s));
            }
        }
        return;
    }

    // ---------------- consumers ----------------
    const u32 gid = threadIdx.x / GTHREADS, tg = threadIdx.x - gid * GTHREADS;
    u32 q = 0, ui = 0;
#ifdef P3GPU_NTT_PROFILE
    u32 kk = 0;   // tiles taken by this group; 8 slots per (CTA, group, tile < 16): smid, t_start, t_full, t_step1, t_step2
#define P3_GSTAMP(slot) do { if (a.prof && tg == 0 && kk < 16) { unsigned long long ts_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ts_)); \
        a.prof[(((size_t)blockIdx.x * NGROUP + gid) * 16 + kk) * 8 + (slot)] = ts_; } } while (0)
#else
#define P3_GSTAMP(slot) do { } while (0)
#endif
    for (u32 it = blockIdx.x; it < a.n_items; it += gridDim.x, ui++) {
        u32 coset, L, T, ct0, ct1;
        decode(it, coset, L, T, ct0, ct1);
        const u32 b = ui & 1u, ph = (ui >> 1) & 1u;
        const uint2 *tws = tws0 + b * R;
        const u32 ibase = (a.l0 == 0 ? 0u : (T << (a.log_n - a.l0))) | L;
        bool tw_ready = false;
        for (u32 ct = ct0; ct < ct1; ct++, q++) {
            const u32 s = q % NSTAGE, k = q / NSTAGE;
            const u32 col = ct * CT, cw = min(CT, a.wc - col);
            u32 *data = stages + (size_t)s * STAGE_WORDS;
            P3_GSTAMP(1);
            // EVERY group waits for EVERY tile and twiddle buffer in sequence order, also those it does not process, and only then
            // lets the ring advance (empty[s] / twempty[b] count all consumer threads).  A parity wait can only tell the current
            // mbarrier phase from the one before it; a group that skipped a stage's previous use could otherwise run ahead of a
            // load that is still in flight and take the older phase for the one it wants (seen with 128-row tiles, which are
            // processed faster than HBM latency varies: corrupted arrival counts, i.e. hangs and mbarrier traps).
            mbar_wait(full_bar(s), k & 1u);
            if (!tw_ready) { mbar_wait(twfull_bar(b), ph); tw_ready = true; }
            if (q % NGROUP != gid) {
                mbar_arrive(empty_bar(s));
                mbar_arrive(twempty_bar(b));
                continue;
            }
            P3_GSTAMP(2);
            const u32 dg = GTHREADS / cw, dc = GTHREADS - dg * cw;
            // ---- step 1 (in place): E1 values per item, Q1 layers
            {
                u32 g = tg / cw, c = tg - g * cw;
                for (; g < E2; ) {
                    u32 x[E1];
                    if (!PERM) {
                        u32 *sp = data + g * CT + c;           // local rows g + m*E2
#pragma unroll
                        for (u32 m = 0; m < E1; m++) x[m] = sp[m * gstride];
                        if (a.has_scale) {
#pragma unroll
                            for (u32 m = 0; m < E1; m++) x[m] = shoup_mul<F>(x[m], a.scale);
                        }
                        reg_network<F, Q1>(x, tws, 1u);
#pragma unroll
                        for (u32 m = 0; m < E1; m++) sp[m * gstride] = x[m];
                    } else {
                        u32 *sp = data + g * gstride + c;      // g = gamma: local rows bitrev_Q2(gamma) + m*E2 sit in group gamma
#pragma unroll
                        for (u32 m = 0; m < E1; m++) x[m] = sp[brev_const<Q1>(m) * CT];
                        if (a.has_scale) {
#pragma unroll
                            for (u32 m = 0; m < E1; m++) x[m] = shoup_mul<F>(x[m], a.scale);
                        }
                        reg_network<F, Q1>(x, tws, 1u);
#pragma unroll
                        for (u32 m = 0; m < E1; m++) sp[brev_const<Q1>(m) * CT] = x[m];
                    }
                    c += dc; g += dg;
                    if (c >= cw) { c -= cw; g++; }
                }
            }
            asm volatile("bar.sync %0, %1;" ::"r"(gid + 1u), "r"((u32)GTHREADS) : "memory");
            P3_GSTAMP(3);
            // ---- step 2: E2 values per item, Q2 layers, results straight to global memory
            {
                // dense output: row pitch w, this tile at column col of coset block `coset`;
                // tiled output: 8-column matrix number ct * n_cosets + coset, row pitch 8
                const u32 ow = a.out_tiled ? CT : a.w;
                u32 *out = a.out_tiled ? a.out + ((((size_t)ct * a.n_cosets + coset) << a.log_n) << 3) : a.out + (size_t)coset * a.out_stride + col;
                const size_t sstride = ((size_t)(a.out_bitrev ? (1u << (a.l0 + Q1)) : (1u << lowbits)) << a.out_sh) * ow;
                u32 g = tg / cw, c = tg - g * cw;
                bool released = false;
                for (; g < E1; ) {
                    u32 x[E2];
                    u32 gg;   // item = local rows gg*E2 + m
                    if (!PERM) {
                        gg = g;
                        const u32 *sp = data + g * gstride + c;
#pragma unroll
                        for (u32 m = 0; m < E2; m++) x[m] = sp[m * CT];
                    } else {
                        gg = __brev(g) >> (32 - Q1);
                        const u32 *sp = data + g * CT + c;
#pragma unroll
                        for (u32 m = 0; m < E2; m++) x[m] = sp[brev_const<Q2>(m) * gstride];
                    }
                    u32 gn = g + dg, cn = c + dc;
                    if (cn >= cw) { cn -= cw; gn++; }
                    if (gn >= E1) {   // last shared-memory read of this thread for this stage: hand it back to the producer
                        fence_proxy_async_smem();
                        mbar_arrive(empty_bar(s));
                        released = true;
                    }
                    reg_network<F, Q2>(x, tws, E1 + gg);
                    if (a.final_reduce) {
#pragma unroll
                        for (u32 m = 0; m < E2; m++) x[m] = fp_reduce<F>(x[m]);
                    }
                    const u32 i0 = ibase | (gg << (lowbits + Q2));
                    const u32 row0 = ((a.out_bitrev ? (__brev(i0) >> brsh) : i0) << a.out_sh) + a.out_add;
                    u32 *p = out + (size_t)row0 * ow + c;
                    if (a.shard_log_rows) {   // peer-memory row sharding (dense, natural network order: a tile's rows are contiguous)
                        const u32 grow = (coset << a.log_n) + row0;
                        p = a.shard_out[grow >> a.shard_log_rows] + (size_t)(grow & ((1u << a.shard_log_rows) - 1u)) * ow + col + c;
                    }
                    if (a.out_bitrev) {
#pragma unroll
                        for (u32 m = 0; m < E2; m++) p[brev_const<Q2>(m) * sstride] = x[m];
                    } else {
#pragma unroll
                        for (u32 m = 0; m < E2; m++) p[m * sstride] = x[m];
                    }
                    g = gn; c = cn;
                }
                if (!released) {   // threads without a step-2 item (ragged tile)
                    fence_proxy_async_smem();
                    mbar_arrive(empty_bar(s));
                }
            }
            mbar_arrive(twempty_bar(b));
            P3_GSTAMP(4);
#ifdef P3GPU_NTT_PROFILE
            kk++;
#endif
        }
    }
}

// ---- twiddle heaps ---------------------------------------------------------------------------
struct TwGenArgs {
    u32 sigma[32];  // sigma[l] = shift^(N/2^(l+1)), Montgomery
    u32 roots[32];  // roots[k] = primitive 2^k-th root (or its inverse), Montgomery
};
template <int F> __global__ void gen_twiddle_heap(uint2 *Z, int log_n, const TwGenArgs a) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= ((size_t)1 << log_n)) return;
    if (idx == 0) { Z[0] = make_uint2(0, 0); return; }
    const int l = 63 - __clzll((long long)idx);
    const u32 q = (u32)(idx - ((size_t)1 << l));
    u32 z = a.sigma[l];
    for (int b = 0; b < l; b++)
        if ((q >> b) & 1u) z = mont_mul<F>(z, a.roots[b + 2]);
    Z[idx] = shoup_pair<F>(from_monty<F>(z));
}

// row i *= base^i  (dft/src/util.rs:32-55 coset_shift_cols), used by coset_idft_batch only
struct PowArgs { u32 pw[32]; };  // pw[k] = base^(2^k), Montgomery
template <int F> __global__ void scale_rows_by_powers(u32 *m, size_t h, size_t w, const PowArgs a) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= h * w) return;
    size_t row = idx / w;
    u32 s = Fp<F>::ONE;
    for (int k = 0; row; k++, row >>= 1)
        if (row & 1) s = mont_mul<F>(s, a.pw[k]);
    m[idx] = mont_mul<F>(m[idx], s);
}
__global__ void broadcast_row(const u32 *in, u32 *out, size_t rows, size_t w) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < rows * w) out[idx] = in[idx % w];
}

// Heap(s) for the size-2^log_n network.  added_bits = 0: one heap for (shift, inverse).  added_bits > 0 (LDE): 2^added_bits
// heaps back to back, block cb for the coset shift * g_big^bitrev(cb).
template <int F>
static int32_t get_twiddles(p3gpu_ctx *ctx, int log_n, int added_bits, u32 shift, int inverse, const uint2 **out) {
    TwiddleKey key{F, log_n, shift, inverse + 2 * added_bits};
    std::lock_guard<std::recursive_mutex> g(ctx->call_mu);   // entry points already hold it; kept for internal callers
    {
        auto it = ctx->twiddles.find(key);
        if (it != ctx->twiddles.end()) { it->second.last_use = ctx->tick; *out = it->second.ptr; return P3GPU_OK; }
    }
    const size_t N = (size_t)1 << log_n, n_cosets = (size_t)1 << added_bits;
    const size_t bytes = n_cosets * N * sizeof(uint2);
    // bounded cache (the reference's map grows without bound; a long-lived prover with many shifts/sizes must not): evict
    // least-recently-used heaps that no call of the current entry point has touched until the new heap fits
    while (ctx->twiddle_bytes + bytes > ctx->twiddle_cap_bytes) {
        auto victim = ctx->twiddles.end();
        for (auto it = ctx->twiddles.begin(); it != ctx->twiddles.end(); ++it)
            if (it->second.last_use < ctx->tick && (victim == ctx->twiddles.end() || it->second.last_use < victim->second.last_use)) victim = it;
        if (victim == ctx->twiddles.end()) break;          // everything left is in use by this call: exceed the cap rather than fail
        P3_CUDA(cudaStreamSynchronize(ctx->stream));       // queued kernels may still read the heap
        P3_CUDA(cudaFree(victim->second.ptr));
        ctx->twiddle_bytes -= victim->second.bytes;
        ctx->twiddles.erase(victim);
    }
    uint2 *Z = nullptr;
    {
        cudaError_t e = cudaMalloc(&Z, bytes);
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu) for a twiddle heap failed: %s", bytes, cudaGetErrorString(e)); cudaGetLastError(); return P3GPU_ENOMEM; }
    }
    const u32 g_big = two_adic_generator<F>((u32)(log_n + added_bits));
    for (size_t cb = 0; cb < n_cosets; cb++) {
        size_t c = 0;
        for (int b = 0; b < added_bits; b++) c |= ((cb >> b) & 1) << (added_bits - 1 - b);
        const u32 s = mont_mul<F>(shift, fp_pow<F>(g_big, c));
        TwGenArgs a;
        for (int l = 0; l < 32; l++) { a.sigma[l] = Fp<F>::ONE; a.roots[l] = Fp<F>::ONE; }
        for (int l = 0; l < log_n; l++) a.sigma[l] = fp_pow<F>(s, (u64)(N >> (l + 1)));
        for (u32 k = 0; k <= (u32)log_n && k <= Fp<F>::TWO_ADICITY; k++) {
            u32 gk = two_adic_generator<F>(k);
            a.roots[k] = inverse ? fp_inv<F>(gk) : gk;
        }
        const unsigned blocks = (unsigned)((N + 255) / 256);
        gen_twiddle_heap<F><<<blocks, 256, 0, ctx->stream>>>(Z + cb * N, log_n, a);
        ctx->launches++;
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { cudaFree(Z); set_error("gen_twiddle_heap launch failed: %s", cudaGetErrorString(e)); return P3GPU_ECUDA; }
    }
    ctx->twiddles.emplace(key, TwiddleEntry{Z, bytes, ctx->tick});
    ctx->twiddle_bytes += bytes;
    *out = Z;
    return P3GPU_OK;
}

// Kernel KERN's dynamic shared-memory limit (at least the default 48 KB) for launches of `smem` bytes, set on ctx's device when
// the previous launch of KERN there asked for another size.  *changed (if given) says so, for whatever the caller derives from
// the size.
template <auto KERN> static int32_t set_smem_limit(p3gpu_ctx *ctx, size_t smem, bool *changed = nullptr) {
    static size_t set[64] = {0};   // per instance and device
    size_t &last = set[ctx->device & 63];
    if (changed) *changed = smem != last;
    if (smem != last) {
        P3_CUDA(cudaFuncSetAttribute(KERN, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, 48 * 1024)));
        last = smem;
    }
    return P3GPU_OK;
}

// Grid of persistent kernel KERN over `items` work items: as many CTAs of `block` threads and `smem` bytes per SM as the register
// file, shared memory (227 KB, 1 KB reserved per CTA) and `cap` allow, at least one, and no more CTAs than items.
template <auto KERN> static int32_t persistent_grid(p3gpu_ctx *ctx, size_t block, size_t smem, size_t cap, size_t items, size_t *grid) {
    static int num_regs = 0;   // per instance; benign race (same value)
    if (num_regs == 0) {
        cudaFuncAttributes fa;
        P3_CUDA(cudaFuncGetAttributes(&fa, KERN));
        num_regs = std::max(fa.numRegs, 16);
    }
    const size_t per_sm = std::min({cap, (227 * 1024) / (smem + 1024), 65536 / (block * (size_t)num_regs)});
    *grid = std::min(items, std::max<size_t>(per_sm, 1) * (size_t)ctx->sm_count);
    return P3GPU_OK;
}

template <int F, int LOG_CT, bool VEC>
static int32_t launch_pass_ct(p3gpu_ctx *ctx, const PassArgs &a) {
    constexpr int THREADS = 256;
    const int r = a.l1 - a.l0;
    const size_t smem = (((size_t)1 << r) << LOG_CT) * 4 + ((size_t)1 << r) * sizeof(uint2);
    constexpr auto kern = ntt_pass_kernel<F, LOG_CT, THREADS, VEC>;
    P3_TRY(set_smem_limit<kern>(ctx, smem));
    const size_t tiles = ((size_t)1 << (a.log_n - r)) * a.n_ctiles * a.n_cosets;
    P3_CHECK(tiles < (1ull << 31), P3GPU_EINVAL, "ntt: grid too large");
    kern<<<(unsigned)tiles, THREADS, smem, ctx->stream>>>(a);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

static int32_t make_pass_tensor_map(const PassArgs &a, const u32 *base, bool tiled, size_t blk_stride, u32 box_w, bool perm, int gs_log,
                                    CUtensorMap *tm);

template <int F, int R_LOG, int CT_T, int THREADS, int NBUF>
static int32_t launch_fast_rct(p3gpu_ctx *ctx, PassArgs a) {
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    const u32 ct = a.ct;
    const u32 e2 = 1u << Q2, e1 = 1u << Q1;
    const u32 padw = (ct + 32u - ((e2 * ct) & 31u)) & 31u;
    const size_t buf_words = ((size_t)e1 * (e2 * ct + padw) + 3) & ~(size_t)3;
    CUtensorMap omap;
    memset(&omap, 0, sizeof omap);
    a.tma_store = a.tma_store && NBUF == 2 && a.vec16;
    if (a.tma_store) {   // the padded tile is the store box: group stride (2^Q2 + 1) * ct words (always so for ct % 4 == 0)
        P3_CHECK(e2 * ct + padw == (e2 + 1) * ct && !a.out_bitrev && a.out_sh == 0 && a.out_add == 0, P3GPU_EINVAL, "ntt: tile layout is no TMA box");
        P3_TRY(make_pass_tensor_map(a, a.out, false, a.out_stride, ct, false, Q2, &omap));
    }
    const size_t smem = NBUF * buf_words * 4 + NBUF * ((size_t)1 << R_LOG) * sizeof(uint2);
    constexpr auto kern = ntt_pass_fast_kernel<F, R_LOG, CT_T, THREADS, NBUF>;
    P3_CHECK(smem <= 227 * 1024, P3GPU_EINVAL, "ntt: tile does not fit shared memory");
    P3_TRY(set_smem_limit<kern>(ctx, smem));
    const size_t tiles = ((size_t)1 << (a.log_n - R_LOG)) * a.n_ctiles * a.n_cosets;
    P3_CHECK(tiles < (1ull << 31), P3GPU_EINVAL, "ntt: grid too large");
    // persistent grid: one CTA per SM (more when the tile is small enough for several to be resident)
    size_t grid;
    P3_TRY(persistent_grid<kern>(ctx, THREADS, smem, NBUF == 1 ? 2048 / THREADS : 2, tiles, &grid));
    kern<<<(unsigned)grid, THREADS, smem, ctx->stream>>>(a, omap);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}
template <int F, int R_LOG, int CT_T>
static int32_t launch_fast_rc(p3gpu_ctx *ctx, const PassArgs &a) {
    static const int threads = env_int("P3GPU_NTT_THREADS", 512);
    if (threads == 256) return launch_fast_rct<F, R_LOG, CT_T, 256, 1>(ctx, a);   // 2-3 single-buffered CTAs per SM
    // default: 1 double-buffered 512-thread CTA per SM.  Measured on H100 (400 W), KoalaBear LDE with blowup 2, ms:
    // 2^20 x 100: 3.58 vs 4.65 for 256 single-buffered threads; 2^20 x 1312: 35.7 vs 40.4.
    return launch_fast_rct<F, R_LOG, CT_T, 512, 2>(ctx, a);
}
template <int F, int R_LOG>
static int32_t launch_fast_r(p3gpu_ctx *ctx, const PassArgs &a) {
    switch (a.ct) {   // compile-time widths keep every shared-memory offset an immediate
        case 16: return launch_fast_rc<F, R_LOG, 16>(ctx, a);
        case 20: return launch_fast_rc<F, R_LOG, 20>(ctx, a);
        case 24: return launch_fast_rc<F, R_LOG, 24>(ctx, a);
        default: return launch_fast_rc<F, R_LOG, 0>(ctx, a);
    }
}
template <int F>
static int32_t launch_fast(p3gpu_ctx *ctx, const PassArgs &a) {
    switch (a.l1 - a.l0) {
        case 6: return launch_fast_r<F, 6>(ctx, a);
        case 7: return launch_fast_r<F, 7>(ctx, a);
        case 8: return launch_fast_r<F, 8>(ctx, a);
        case 9: return launch_fast_r<F, 9>(ctx, a);
        default: return launch_fast_r<F, 10>(ctx, a);
    }
}

// Cluster size of the band pass: clusters of 8 CTAs fill 120 of the H100's 132 SMs, as clusters of 4 do, and stream at the same
// rate (tools/band_probe, DESIGN 4.1).  An eighth of a band is small enough for the 3-slot ring that lets the exchange of one band
// run beside the local steps of another; the price is that 7/8 of each eighth crosses SMs instead of 3/4 of a quarter.
constexpr int BAND_CL = 8;
static bool band_pass_eligible(const PassArgs &a) {
    const int r = a.l1 - a.l0;
    return env_int("P3GPU_NTT_BAND", 1) != 0 && a.l1 == a.log_n && r >= 7 && r <= 10 && a.w % 4 == 0 && a.in_stride % 4 == 0 &&
           a.out_stride % 4 == 0 && ((reinterpret_cast<uintptr_t>(a.in) | reinterpret_cast<uintptr_t>(a.out)) % 16) == 0 &&
           (((size_t)a.w * 4) << r) / BAND_CL <= BAND_SLOT_BYTES;
}
// Widths up to BAND_NARROW_W take ntt_band_pass_narrow_kernel: at 2^20 rows it is the faster one up to 48 columns (0.13 against
// 0.28 ms at 4, 0.41 against 0.50 at 48), the 8-CTA kernel from 64 (0.56 against 0.65 ms) and at every wider shape (DESIGN 4.1).
constexpr u32 BAND_NARROW_W = 48;
static int32_t make_unit_tensor_map(const u32 *base, u32 w, int log_n, int r, u32 rows, CUtensorMap *tm);
// GATHER: a.in is the fused pass's tile-major scratch, read through gmap (make_tile_major_tensor_maps)
template <int F, int R_LOG, bool NARROW, bool STRIDED = false, bool GATHER = false>
static int32_t launch_band_r(p3gpu_ctx *ctx, PassArgs a, const CUtensorMap *gmap = nullptr) {
    static_assert(!(NARROW && STRIDED), "the strided first pass runs in 8-CTA clusters only");
    static_assert(!(NARROW && GATHER), "the gather mode runs in 8-CTA clusters only");
    constexpr int CL = NARROW ? 4 : BAND_CL, SLOTS = NARROW ? 2 : 3;
    const size_t qbytes = (((size_t)a.w * 4) << R_LOG) / CL;
    const size_t tw_bytes = ((size_t)1 << R_LOG) * sizeof(uint2);
    const size_t smem = STRIDED ? 4 * (qbytes + 8) + tw_bytes : SLOTS * (qbytes + tw_bytes + 8);
    constexpr auto kern = [] {
        if constexpr (NARROW) return ntt_band_pass_narrow_kernel<F, R_LOG, CL>;
        else return ntt_band_pass_kernel<F, R_LOG, CL, GATHER, STRIDED>;
    }();
    CUtensorMap imap, omap;
    memset(&imap, 0, sizeof imap); memset(&omap, 0, sizeof omap);
    if constexpr (STRIDED) {
        P3_TRY(make_unit_tensor_map(a.in, a.w, a.log_n, R_LOG, (1u << R_LOG) / CL, &imap));
        P3_TRY(make_unit_tensor_map(a.out, a.w, a.log_n, R_LOG, (1u << R_LOG) / CL, &omap));
    }
    if constexpr (GATHER) {
        P3_CHECK(gmap != nullptr, P3GPU_EINVAL, "ntt: the gather band pass needs its tensor map");
        imap = *gmap;
    }
    // per instantiation and device: the number of clusters that fit at once, for the size set_smem_limit last saw
    static int clusters[64] = {0};
    const int dev = ctx->device & 63;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = CL; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(NARROW ? BAND_NARROW_THREADS : BAND_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = ctx->stream;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    bool changed;
    P3_TRY(set_smem_limit<kern>(ctx, smem, &changed));
    if (changed) {
        cfg.gridDim = dim3(CL * ctx->sm_count);
        int n = 0;
        P3_CUDA(cudaOccupancyMaxActiveClusters(&n, kern, &cfg));
        P3_CHECK(n > 0, P3GPU_ECUDA, "ntt: no %d-CTA cluster of the band pass fits the device", CL);
        clusters[dev] = n;
    }
    const size_t bands = (size_t)a.n_cosets << (a.log_n - R_LOG);
    cfg.gridDim = dim3((unsigned)(CL * std::min<size_t>(bands, (size_t)clusters[dev])));
    if constexpr (NARROW) P3_CUDA(cudaLaunchKernelEx(&cfg, kern, a));
    else P3_CUDA(cudaLaunchKernelEx(&cfg, kern, a, imap, omap));
    ctx->launches++;
    return P3GPU_OK;
}
// gmap != nullptr: the gather mode over the fused pass's tile-major scratch a.in (w > BAND_NARROW_W, see coset_lde_impl)
template <int F>
static int32_t launch_band(p3gpu_ctx *ctx, PassArgs a, const CUtensorMap *gmap = nullptr) {
    // profiling build only: NOLOAD / NOSTORE skip the part's bulk copies, NOBFLY bit 0 steps A and B, bit 1 the exchange
    a.skip_bfly = env_int("P3GPU_NTT_NOBFLY", 0);
    a.skip_load = env_int("P3GPU_NTT_NOLOAD", 0); a.skip_store = env_int("P3GPU_NTT_NOSTORE", 0);
    const bool narrow = a.w <= BAND_NARROW_W;
    if (gmap) {
        P3_CHECK(!narrow, P3GPU_EINVAL, "ntt: the gather band pass needs more than %u columns", BAND_NARROW_W);
        switch (a.l1 - a.l0) {
            case 7: return launch_band_r<F, 7, false, false, true>(ctx, a, gmap);
            case 8: return launch_band_r<F, 8, false, false, true>(ctx, a, gmap);
            case 9: return launch_band_r<F, 9, false, false, true>(ctx, a, gmap);
            default: return launch_band_r<F, 10, false, false, true>(ctx, a, gmap);
        }
    }
    switch (a.l1 - a.l0) {
        case 7: return narrow ? launch_band_r<F, 7, true>(ctx, a) : launch_band_r<F, 7, false>(ctx, a);
        case 8: return narrow ? launch_band_r<F, 8, true>(ctx, a) : launch_band_r<F, 8, false>(ctx, a);
        case 9: return narrow ? launch_band_r<F, 9, true>(ctx, a) : launch_band_r<F, 9, false>(ctx, a);
        default: return narrow ? launch_band_r<F, 10, true>(ctx, a) : launch_band_r<F, 10, false>(ctx, a);
    }
}

// The first pass of a network (l0 = 0, r = l1 layers) on strided units (ntt_band_pass_kernel<..., STRIDED>): one block, no pitch, a
// part (2^r / 8 rows of w words) that fits a ring slot, and w within the 256-element tensor box; P3GPU_NTT_BAND=0 keeps the tile
// kernel.  Below BAND_FIRST_MIN_W columns the tile kernel is the faster one, or no gain was measured (DESIGN 4.1).
constexpr u32 BAND_FIRST_MIN_W = 100;
static bool band_first_pass_eligible(const PassArgs &a) {
    const int r = a.l1 - a.l0;
    return env_int("P3GPU_NTT_BAND", 1) != 0 && a.l0 == 0 && r >= 7 && r <= 10 && a.n_cosets <= 1 && a.in_stride == 0 &&
           a.out_stride == 0 && !a.in_bitrev && !a.out_bitrev && a.out_sh == 0 && a.out_add == 0 && a.w % 4 == 0 &&
           a.w >= BAND_FIRST_MIN_W && a.w <= 256 && ((reinterpret_cast<uintptr_t>(a.in) | reinterpret_cast<uintptr_t>(a.out)) % 16) == 0 &&
           (((size_t)a.w * 4) << r) / BAND_CL <= BAND_SLOT_BYTES;
}
template <int F>
static int32_t launch_band_first(p3gpu_ctx *ctx, PassArgs a) {
    a.n_cosets = 1;
    a.skip_bfly = env_int("P3GPU_NTT_NOBFLY", 0);
    a.skip_load = env_int("P3GPU_NTT_NOLOAD", 0); a.skip_store = env_int("P3GPU_NTT_NOSTORE", 0);
    switch (a.l1) {
        case 7: return launch_band_r<F, 7, false, true>(ctx, a);
        case 8: return launch_band_r<F, 8, false, true>(ctx, a);
        case 9: return launch_band_r<F, 9, false, true>(ctx, a);
        default: return launch_band_r<F, 10, false, true>(ctx, a);
    }
}

// Instances of the fused kernel that have a producer-warp form: every one but the runtime-width instance at r = 10, whose 384
// consumer threads need 168 registers against the 152 that 416 threads leave them.
template <int R_LOG, int CT_T> constexpr bool lde_mid_producer() { return R_LOG < 10 || CT_T != 0; }

template <int F, int R_LOG, bool TILES, int CT_T, bool PROD>
static int32_t launch_lde_mid_rcp(p3gpu_ctx *ctx, const PassArgs &a, const uint2 *tw_fwd, const CUtensorMap &omap, const CUtensorMap &imap) {
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    constexpr int THREADS = lde_mid_threads<R_LOG, CT_T>(), BLOCK = THREADS + (PROD ? 32 : 0);
    const size_t ct = a.ct, e1 = (size_t)1 << Q1, e2 = (size_t)1 << Q2;
    const size_t gs1 = e2 * ct + ((ct + 32 - ((e2 * ct) & 31)) & 31), gs2 = e1 * ct + ((ct + 32 - ((e1 * ct) & 31)) & 31);
    const size_t buf_words = (std::max(e1 * gs1, e2 * gs2) + 3) & ~(size_t)3;
    const size_t smem = 2 * buf_words * 4 + (2 + a.n_cosets) * ((size_t)1 << R_LOG) * sizeof(uint2) + (PROD ? 5 * 8 : 0);
    P3_CHECK(smem <= 227 * 1024, P3GPU_EINVAL, "ntt: fused LDE tile does not fit shared memory");
    P3_CHECK(gs2 == (e1 + 1) * ct && gs1 == (e2 + 1) * ct, P3GPU_EINVAL, "ntt: fused LDE tile layout is no TMA box");
    constexpr auto kern = ntt_lde_mid_kernel<F, R_LOG, TILES, CT_T, PROD>;
    P3_TRY(set_smem_limit<kern>(ctx, smem));
    const size_t tiles = ((size_t)1 << (a.log_n - R_LOG)) * a.n_ctiles;
    // persistent grid: as many CTAs per SM as threads, registers and shared memory allow (one at 2^20 rows)
    size_t grid;
    P3_TRY(persistent_grid<kern>(ctx, BLOCK, smem, 2048 / BLOCK, tiles, &grid));
    kern<<<(unsigned)grid, BLOCK, smem, ctx->stream>>>(a, tw_fwd, omap, imap);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}
template <int F, int R_LOG, bool TILES, int CT_T>
static int32_t launch_lde_mid_rc(p3gpu_ctx *ctx, const PassArgs &a, const uint2 *tw_fwd, const CUtensorMap &omap, const CUtensorMap &imap) {
    if constexpr (lde_mid_producer<R_LOG, CT_T>()) return launch_lde_mid_rcp<F, R_LOG, TILES, CT_T, true>(ctx, a, tw_fwd, omap, imap);
    else return launch_lde_mid_rcp<F, R_LOG, TILES, CT_T, false>(ctx, a, tw_fwd, omap, imap);
}
template <int F, int R_LOG, bool TILES>
static int32_t launch_lde_mid_rt(p3gpu_ctx *ctx, const PassArgs &a, const uint2 *tw_fwd, const CUtensorMap &omap, const CUtensorMap &imap) {
    switch (a.ct) {
        case 16: return launch_lde_mid_rc<F, R_LOG, TILES, 16>(ctx, a, tw_fwd, omap, imap);
        case 20: return launch_lde_mid_rc<F, R_LOG, TILES, 20>(ctx, a, tw_fwd, omap, imap);
        default: return launch_lde_mid_rc<F, R_LOG, TILES, 0>(ctx, a, tw_fwd, omap, imap);
    }
}
template <int F, int R_LOG>
static int32_t launch_lde_mid_r(p3gpu_ctx *ctx, const PassArgs &a, bool tiles, const uint2 *tw_fwd, const CUtensorMap &omap,
                                const CUtensorMap &imap) {
    return tiles ? launch_lde_mid_rt<F, R_LOG, true>(ctx, a, tw_fwd, omap, imap) : launch_lde_mid_rt<F, R_LOG, false>(ctx, a, tw_fwd, omap, imap);
}

// ---- pipelined kernel: host side -------------------------------------------------------------------------------
typedef CUresult (*TensorMapEncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                      const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                      CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TensorMapEncodeFn tensor_map_encoder() {
    static TensorMapEncodeFn fn = []() -> TensorMapEncodeFn {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess)
            return nullptr;
        return reinterpret_cast<TensorMapEncodeFn>(p);
    }();
    return fn;
}

// 5-D view of a pass's input or output over `base` for tensor copies of whole tiles: (column, row-in-group, group, L, T) with
// the tile's local row rho = group * 2^gs_log + row-in-group at global row  T * 2^(n-l0) + rho * 2^lowbits + L   (PERM: block * 2^r
// + position).  The box is (box_w, 2^gs_log + 1, 2^(r - gs_log), 1, 1): one row more per group than the tensor has, which a load
// zero-fills and a store skips, so the box is exactly the padded shared-memory tile (group stride (2^gs_log + 1) * box_w words).
// box_w * 4 must be a multiple of 16 bytes; columns past the width are skipped by stores (a ragged last column tile).
// Dense layout (tiled = 0): pitch w; blk_stride != 0 (= w * 2^n) stacks the n_cosets blocks in the last dimension, whose
// coordinate is then T + (block << l0).  Tiled layout (ntt_pass_pipe_kernel only): 8-column matrices of 2^n rows.
static int32_t make_pass_tensor_map(const PassArgs &a, const u32 *base, bool tiled, size_t blk_stride, u32 box_w, bool perm, int gs_log,
                                    CUtensorMap *tm) {
    TensorMapEncodeFn enc = tensor_map_encoder();
    P3_CHECK(enc != nullptr, P3GPU_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const int r = a.l1 - a.l0, lowbits = a.log_n - a.l1;
    const u32 wc = a.wc ? a.wc : a.w;
    const cuuint64_t pitch = tiled ? 32 : (cuuint64_t)a.w * 4;
    const cuuint64_t n_ctiles = (wc + 7) / 8;
    cuuint64_t dims[5], strides[4];
    cuuint32_t box[5] = {box_w, (1u << gs_log) + 1, 1u << (r - gs_log), 1, 1}, es[5] = {1, 1, 1, 1, 1};
    dims[0] = tiled ? 8 : wc;
    dims[1] = 1ull << gs_log; dims[2] = 1ull << (r - gs_log);
    const cuuint64_t blocks = tiled ? n_ctiles * a.in_blocks : (blk_stride ? a.n_cosets : 1);
    if (!perm) {
        dims[3] = 1ull << lowbits; dims[4] = blocks << a.l0;
        strides[0] = pitch << lowbits; strides[1] = pitch << (lowbits + gs_log); strides[2] = pitch; strides[3] = pitch << (a.log_n - a.l0);
    } else {
        dims[3] = 1; dims[4] = blocks << (a.log_n - r);
        strides[0] = pitch; strides[1] = pitch << gs_log; strides[2] = pitch; strides[3] = pitch << r;
    }
    const CUresult rc = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 5, const_cast<u32 *>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    P3_CHECK(rc == CUDA_SUCCESS, P3GPU_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)rc);
    return P3GPU_OK;
}

// 3-D view of one dense 2^log_n x w block for the strided band pass: (column, unit L, i) at row L + 2^(log_n - r) * i; the box
// (w, 1, rows) is one part, `rows` dense rows of w words in shared memory.  w % 4 == 0, w <= 256, base 16-byte aligned.
static int32_t make_unit_tensor_map(const u32 *base, u32 w, int log_n, int r, u32 rows, CUtensorMap *tm) {
    TensorMapEncodeFn enc = tensor_map_encoder();
    P3_CHECK(enc != nullptr, P3GPU_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t pitch = (cuuint64_t)w * 4;
    cuuint64_t dims[3] = {w, 1ull << (log_n - r), 1ull << r}, strides[2] = {pitch, pitch << (log_n - r)};
    cuuint32_t box[3] = {w, 1, rows}, es[3] = {1, 1, 1};
    const CUresult rc = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<u32 *>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    P3_CHECK(rc == CUDA_SUCCESS, P3GPU_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)rc);
    return P3GPU_OK;
}

// The tile-major scratch between the fused LDE pass and the gathering last pass (2^2r rows of w = n_ct * ct columns, n_cosets
// cosets).  Coset cs's forward tile L and column tile c make tile tt = L * n_ct + c, whose result is ONE dense block of 2^r rows x ct
// words at word offset ((cs * 2^r + L) * n_ct + c) * 2^r * ct.  Forward step 2's local row i = j * 2^Q1 + b holds what goes to row
// L + 2^r * i of the coset block, and is block row tile_block_row(i) = b * 2^Q2 + j: the order in which ntt_lde_mid_kernel<..., TILES,
// ...> stores each warp's register b as one whole 128-byte line (ct % 4 == 0, so 2^Q2 * ct words are a multiple of 32).  Row L of
// band i is block row tile_block_row(i) of tiles L * n_ct .. L * n_ct + n_ct - 1, so the last pass gathers each row of its part from
// n_ct blocks instead of reading one contiguous run.  The gather map (ntt_band_pass_kernel<..., GATHER>) is (column, column tile,
// block row, tile row L, coset) with box (ct, n_ct, 1, rows, 1): rows L .. L + rows - 1 of band i, w words each, land row-major as
// one part.
static int32_t make_tile_major_tensor_maps(const u32 *base, u32 ct, u32 n_ct, int r, u32 n_cosets, u32 rows, CUtensorMap *gather_map) {
    TensorMapEncodeFn enc = tensor_map_encoder();
    P3_CHECK(enc != nullptr, P3GPU_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t seg = (cuuint64_t)ct * 4, blk = seg << r, tile_row = blk * n_ct, coset = tile_row << r;
    const cuuint64_t dims[5] = {ct, n_ct, 1ull << r, 1ull << r, n_cosets};
    const cuuint64_t strides[4] = {blk, seg, tile_row, coset};
    const cuuint32_t box[5] = {ct, n_ct, 1, rows, 1}, es[5] = {1, 1, 1, 1, 1};
    const CUresult rc = enc(gather_map, CU_TENSOR_MAP_DATA_TYPE_UINT32, 5, const_cast<u32 *>(base), dims, strides, box, es,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    P3_CHECK(rc == CUDA_SUCCESS, P3GPU_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)rc);
    return P3GPU_OK;
}

// P3GPU_NTT_PIPE (read per call: the tests switch between the kernel families): 1 = TMA pipeline for every eligible pass and
// the tiled LDE for every eligible LDE, 0 = never, unset (-1) = the H100 choice: dense passes of 10 layers on the cp.async
// kernel, everything else eligible on the pipeline.  Measured on H100 (400 W), ms, cp.async kernel (512 threads) vs pipeline
// (tiled intermediates for the LDE), blowup 2: LDE KoalaBear 2^20 x 100 3.3 vs 4.0, 2^20 x 1312 35.4 vs 36.5, BabyBear
// 2^22 x 300 85 vs 62, 2^21 x 200 24.3 vs 24.1, KoalaBear 2^18 x 64 0.45 vs 0.37; DFT 2^20 x 100 1.39 vs 2.36, 2^21 x 200
// 8.5 vs 6.6.  (2^22 and 2^21 run 8+7+7 and 7+7+7 layers, 2^18 9+9.)  Those LDE figures are for four launches; the cp.async
// LDE now fuses its middle passes and stores tiles with tensor copies (coset_lde_impl): 2.72 ms for 2^20 x 100 (DESIGN 4.1).
static int pipe_mode() { return env_int("P3GPU_NTT_PIPE", -1); }
static bool cp_async_pass(int r) { return r == 10; }

static bool pipe_eligible(const PassArgs &a) {
    const int mode = pipe_mode();
    if (mode == 0) return false;
    const int r = a.l1 - a.l0;
    if (r < 6 || r > 10) return false;
    if (a.in_tiled || a.out_tiled) return true;                                 // set up by lde_tiled_impl, which checked
    if (mode != 1 && cp_async_pass(r)) return false;
    if (a.w % 4 != 0 || a.w < 8 || a.w > 8192) return false;                    // TMA: 16-byte global strides; mbarrier count per unit
    if (reinterpret_cast<uintptr_t>(a.in) % 16 != 0) return false;
    if ((((size_t)a.w * 4) << a.log_n) >= (1ull << 40)) return false;           // TMA stride limit
    if (a.in_stride != 0 && a.in_stride != ((size_t)a.w << a.log_n)) return false;
    if (a.in_bitrev && (a.l0 != 0 || (a.in_stride != 0 && a.n_cosets > 1))) return false;
    return true;
}

template <int F, int R_LOG, bool PERM>
static int32_t launch_pipe_r(p3gpu_ctx *ctx, PassArgs a) {
    constexpr int NSTAGE = 6, NGROUP = 4, GTHREADS = 128;
    constexpr int Q2 = (R_LOG + 1) / 2, Q1 = R_LOG - Q2;
    constexpr size_t GS = PERM ? (1u << Q1) : (1u << Q2), NG = PERM ? (1u << Q2) : (1u << Q1);
    constexpr size_t box_bytes = NG * (GS + 1) * 8 * 4;
    constexpr size_t smem = NSTAGE * box_bytes + 2 * ((size_t)1 << R_LOG) * sizeof(uint2) + (2 * NSTAGE + 4) * 8;
    static_assert(smem <= 227 * 1024, "pipelined NTT kernel: shared memory budget");
    CUtensorMap tm;
    if (a.wc == 0) a.wc = a.w;
    if (a.in_blocks == 0) a.in_blocks = 1;
    P3_TRY(make_pass_tensor_map(a, a.in, a.in_tiled, a.in_stride, 8, PERM, PERM ? Q1 : Q2, &tm));
    a.n_ctiles = (a.wc + 7) / 8;
    const size_t units = ((size_t)1 << (a.log_n - R_LOG)) * a.n_cosets;
    // few units (small transforms): split a unit's column tiles over several CTAs so that every SM has work
    size_t csplit = units >= 2 * (size_t)ctx->sm_count ? 1 : std::min<size_t>(a.n_ctiles, (2 * (size_t)ctx->sm_count + units - 1) / units);
    a.tpi = (u32)((a.n_ctiles + csplit - 1) / csplit);
    csplit = (a.n_ctiles + a.tpi - 1) / a.tpi;
    a.csplit = (u32)csplit;
    const size_t items = units * csplit;
    P3_CHECK(items < (1ull << 31), P3GPU_EINVAL, "ntt: too many tiles");
    P3_CHECK((size_t)a.tpi * NGROUP * GTHREADS < (1u << 20), P3GPU_EINVAL, "ntt: too many column tiles per unit for the mbarrier count");
    a.n_items = (u32)items;
    constexpr auto kern = ntt_pass_pipe_kernel<F, R_LOG, PERM, NSTAGE, NGROUP, GTHREADS>;
    P3_TRY(set_smem_limit<kern>(ctx, smem));
    const size_t grid = std::min(items, (size_t)ctx->sm_count);
    kern<<<(unsigned)grid, NGROUP * GTHREADS + 32, smem, ctx->stream>>>(tm, a);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}
template <int F, int R_LOG>
static int32_t launch_pipe_p(p3gpu_ctx *ctx, const PassArgs &a) {
    return a.in_bitrev ? launch_pipe_r<F, R_LOG, true>(ctx, a) : launch_pipe_r<F, R_LOG, false>(ctx, a);
}
template <int F>
static int32_t launch_pipe(p3gpu_ctx *ctx, const PassArgs &a) {
    switch (a.l1 - a.l0) {
        case 6: return launch_pipe_p<F, 6>(ctx, a);
        case 7: return launch_pipe_p<F, 7>(ctx, a);
        case 8: return launch_pipe_p<F, 8>(ctx, a);
        case 9: return launch_pipe_p<F, 9>(ctx, a);
        default: return launch_pipe_p<F, 10>(ctx, a);
    }
}

// Column tile width of the fast kernel: all tiles of a launch share one width (a ragged last tile is allowed).
// Prefer exact divisors that keep 16-byte alignment (16, 20, 24 columns = 64/80/96-byte row segments).
static u32 choose_tile_width(u32 w) {
    if (w <= 24) return w;
    static const int forced = env_int("P3GPU_NTT_CT", 0);
    if (forced) return (u32)forced;
    for (u32 ct : {16u, 20u, 24u, 12u})
        if (w % ct == 0) return ct;
    const u32 n = (w + 19) / 20;                 // ~20 columns per tile, nearly equal tiles
    u32 ct = (w + n - 1) / n;
    ct = (ct + 3) & ~3u;
    return ct > 24 ? 24 : ct;
}

// Column tile width of the fused LDE middle pass: at most 20 columns (24-column tiles become two of 12); 0 = no 16-byte
// aligned width (w % 4 != 0), which the fused pass does not take.
static u32 lde_mid_tile_width(u32 w) {
    const u32 ct = choose_tile_width(w);
    if (w % 4 != 0 || ct % 4 != 0 || ct > 24) return 0;
    return ct == 24 ? 12 : ct;
}

// a: the inverse network's second pass (l0 = r, l1 = 2r) over the coefficient buffer, writing the forward networks' first-pass
// results of a.n_cosets cosets to a.out (blocks a.out_stride apart); tw_fwd: the cosets' forward heaps, a.tw_stride apart.
// tiles: a.out is the tile-major scratch instead (make_tile_major_tensor_maps), one dense block per tile, stored from registers.
template <int F>
static int32_t launch_lde_mid(p3gpu_ctx *ctx, PassArgs a, const uint2 *tw_fwd, bool tiles = false) {
    a.ct = lde_mid_tile_width(a.w);
    a.n_ctiles = (a.w + a.ct - 1) / a.ct;
    a.prof = prof_window();
    a.skip_bfly = env_int("P3GPU_NTT_NOBFLY", 0); a.skip_store = env_int("P3GPU_NTT_NOSTORE", 0);
    // output = the forward networks' first pass (layers [0, r)) over the cosets' blocks: tile L, local row j*2^Q1 + b at row
    // L + 2^r * (j*2^Q1 + b), i.e. the pass map with groups of 2^Q1 rows (the forward layout gs2 = (2^Q1 + 1) * ct words)
    const int r = a.l1 - a.l0;
    PassArgs o = a;
    o.l0 = 0; o.l1 = r;
    CUtensorMap omap, imap;
    memset(&omap, 0, sizeof omap);
    if (!tiles) P3_TRY(make_pass_tensor_map(o, a.out, false, a.out_stride, a.ct, false, r / 2, &omap));
    // input (producer-warp form): inverse tile T = coefficient rows T * 2^r + rho in the inverse layout, groups of 2^ceil(r/2) rows
    P3_TRY(make_pass_tensor_map(a, a.in, false, 0, a.ct, false, (r + 1) / 2, &imap));
    switch (r) {
        case 7: return launch_lde_mid_r<F, 7>(ctx, a, tiles, tw_fwd, omap, imap);
        case 8: return launch_lde_mid_r<F, 8>(ctx, a, tiles, tw_fwd, omap, imap);
        case 9: return launch_lde_mid_r<F, 9>(ctx, a, tiles, tw_fwd, omap, imap);
        default: return launch_lde_mid_r<F, 10>(ctx, a, tiles, tw_fwd, omap, imap);
    }
}

// One pass over all columns.
//   fast path (7 <= r <= 10): ONE launch, tiles of choose_tile_width(w) columns (16/20/24; ragged last tile allowed).
//   generic path: columns are split greedily into power-of-two tiles of main_ct, main_ct/2, ... columns.
template <int F>
static int32_t launch_pass(p3gpu_ctx *ctx, PassArgs a, unsigned n_cosets, int main_log_ct) {
    a.n_cosets = n_cosets;
    const int r = a.l1 - a.l0;
    a.prof = prof_window();
    if (!env_int("P3GPU_NTT_GENERIC", 0) && pipe_eligible(a)) return launch_pipe<F>(ctx, a);
    if (r >= 6 && r <= 10 && !env_int("P3GPU_NTT_GENERIC", 0)) {
        const u32 ct = choose_tile_width(a.w);
        // 16-byte cp.async / TMA bulk stores need every row segment of every tile 16-byte aligned on both sides
        const bool al16 = (a.w % 4 == 0) && (ct % 4 == 0) &&
                          ((reinterpret_cast<uintptr_t>(a.in) | reinterpret_cast<uintptr_t>(a.out)) % 16 == 0) &&
                          ((a.in_stride | a.out_stride) % 4 == 0);
        a.col0 = 0; a.ct = ct; a.n_ctiles = (a.w + ct - 1) / ct; a.vec16 = al16;
        a.skip_bfly = env_int("P3GPU_NTT_NOBFLY", 0);
        a.skip_load = env_int("P3GPU_NTT_NOLOAD", 0); a.skip_store = env_int("P3GPU_NTT_NOSTORE", 0);
        return launch_fast<F>(ctx, a);
    }
    const bool aligned = (a.w % 4 == 0) && ((reinterpret_cast<uintptr_t>(a.in) | reinterpret_cast<uintptr_t>(a.out)) % 16 == 0) &&
                         ((a.in_stride | a.out_stride) % 4 == 0);
    u32 col = 0, rem = a.w;
    for (int lct = main_log_ct; lct >= 0 && rem; lct--) {
        const u32 ct = 1u << lct;
        const u32 n = rem >> lct;
        if (!n) continue;
        a.col0 = col; a.n_ctiles = n; a.ct = ct;
        const bool vec = aligned && lct >= 2 && (col % 4 == 0);
        int32_t rc;
        switch (lct) {
            case 5: rc = vec ? launch_pass_ct<F, 5, true>(ctx, a) : launch_pass_ct<F, 5, false>(ctx, a); break;
            case 4: rc = vec ? launch_pass_ct<F, 4, true>(ctx, a) : launch_pass_ct<F, 4, false>(ctx, a); break;
            case 3: rc = vec ? launch_pass_ct<F, 3, true>(ctx, a) : launch_pass_ct<F, 3, false>(ctx, a); break;
            case 2: rc = vec ? launch_pass_ct<F, 2, true>(ctx, a) : launch_pass_ct<F, 2, false>(ctx, a); break;
            case 1: rc = launch_pass_ct<F, 1, false>(ctx, a); break;
            default: rc = launch_pass_ct<F, 0, false>(ctx, a); break;
        }
        P3_TRY(rc);
        col += n * ct; rem -= n * ct;
    }
    return P3GPU_OK;
}

struct ShardedOut {
    unsigned world, log_rows;       // ranks; log2 of the rows per rank (LDE height / world)
    u32 *out[16];                   // per rank: its (rows x w_total) row-major block (own memory or an IPC-mapped peer)
    size_t w_total, col_off;        // pitch of those blocks; first column this rank's column block occupies in them
};

struct NetworkPlan {
    int n_passes;
    int bounds[8];  // layer boundaries: pass k covers [bounds[k], bounds[k+1])
};
static NetworkPlan plan_passes(int log_n, int max_r) {
    NetworkPlan p;
    p.n_passes = (log_n + max_r - 1) / max_r;
    if (p.n_passes < 1) p.n_passes = 1;
    int base = log_n / p.n_passes, extra = log_n % p.n_passes;
    p.bounds[0] = 0;
    for (int k = 0; k < p.n_passes; k++) p.bounds[k + 1] = p.bounds[k] + base + (k < extra ? 1 : 0);
    return p;
}
static int network_max_r() { return std::min(12, std::max(4, env_int("P3GPU_NTT_MAXR", 10))); }

// Runs the size-2^log_n network on n_cosets (input, output, twiddle heap) triples laid out at fixed strides.
//   src: input rows, natural order unless in_bitrev (then element i of the network is read from row bitrev(i))
//   dst: output.  Default: network order (row i = network position i).  With out_bitrev / out_sh / out_add the last pass
//        writes position i to row (bitrev(i) << out_sh) + out_add, i.e. natural order (optionally interleaved);
//        that remap cannot run in place, so multi-pass plans then keep intermediate data in tmp (h*w words per coset).
template <int F>
static int32_t run_network(p3gpu_ctx *ctx, int log_n, size_t w, const uint2 *tw, size_t tw_stride, unsigned n_cosets,
                           const u32 *src, size_t src_stride, int in_bitrev, u32 *dst, size_t dst_stride, int out_bitrev,
                           int out_sh, u32 out_add, u32 *tmp, bool has_scale, uint2 scale, bool final_reduce) {
    const int main_log_ct = std::min(5, std::max(0, env_int("P3GPU_NTT_LOGCT", 4)));
    const NetworkPlan plan = plan_passes(log_n, network_max_r());
    const bool remap = out_bitrev || out_sh != 0 || out_add != 0;
    const size_t hw = ((size_t)1 << log_n) * w;
    if (remap && plan.n_passes > 1) P3_CHECK(tmp != nullptr, P3GPU_EINVAL, "ntt: scratch missing");
    for (int k = 0; k < plan.n_passes; k++) {
        PassArgs a;
        memset(&a, 0, sizeof a);
        const bool first = (k == 0), last = (k == plan.n_passes - 1);
        a.w = (u32)w; a.log_n = log_n; a.l0 = plan.bounds[k]; a.l1 = plan.bounds[k + 1];
        a.tw = tw; a.tw_stride = tw_stride;
        u32 *mid = remap ? tmp : dst;
        const size_t mid_stride = remap ? hw : dst_stride;
        a.in = first ? src : mid;
        a.in_stride = first ? src_stride : mid_stride;
        a.in_bitrev = first ? in_bitrev : 0;
        if (last) {
            a.out = dst; a.out_stride = dst_stride;
            a.out_bitrev = out_bitrev; a.out_sh = out_sh; a.out_add = out_add;
            a.final_reduce = final_reduce;
        } else {
            a.out = mid; a.out_stride = mid_stride;
        }
        if (first) { a.has_scale = has_scale; a.scale = scale; }
        P3_TRY(launch_pass<F>(ctx, a, n_cosets, main_log_ct));
    }
    return P3GPU_OK;
}

template <int F> static uint2 inv_height_scale(size_t h) {
    return shoup_pair<F>(from_monty<F>(fp_inv<F>(to_monty<F>((u32)(h % Fp<F>::P)))));
}

template <int F>
static int32_t dft_batch_impl(p3gpu_ctx *ctx, int kind, const u32 *d_in, u32 *d_out, size_t h, size_t w, u32 shift) {
    const int log_n = (int)log2_floor(h);
    if (log_n == 0) {  // size-1 transform is the identity for every kind
        if (d_in != d_out) P3_CUDA(cudaMemcpyAsync(d_out, d_in, w * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        return P3GPU_OK;
    }
    const bool inverse = (kind == P3GPU_IDFT || kind == P3GPU_COSET_IDFT);
    const u32 tw_shift = (kind == P3GPU_COSET_DFT) ? shift : Fp<F>::ONE;
    const uint2 *tw = nullptr;
    P3_TRY(get_twiddles<F>(ctx, log_n, 0, tw_shift, inverse, &tw));
    void *tmp = nullptr;
    P3_TRY(ctx_scratch(ctx, h * w * 4, &tmp));
    P3_TRY(run_network<F>(ctx, log_n, w, tw, 0, 1, d_in, 0, 0, d_out, 0, /*out_bitrev=*/1, 0, 0, (u32 *)tmp, inverse,
                          inverse ? inv_height_scale<F>(h) : make_uint2(0, 0), true));
    if (kind == P3GPU_COSET_IDFT) {  // traits.rs:145-155: coefficient i *= shift^-i
        PowArgs pa;
        u32 b = fp_inv<F>(shift);
        for (int k = 0; k < 32; k++) { pa.pw[k] = b; b = mont_mul<F>(b, b); }
        const size_t n = h * w;
        scale_rows_by_powers<F><<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_out, h, w, pa);
        ctx->launches++;
        P3_CUDA(cudaGetLastError());
    }
    return P3GPU_OK;
}

// coset_lde_batch (bit-reversed output rows) on the pipelined kernel with COLUMN-TILE-MAJOR intermediates.
// Between passes the data lives as one 8-column matrix (32-byte rows) per column tile and coset ("tiled" layout): every
// 32-byte row segment a pass touches is then one aligned DRAM sector, and the contiguous passes stream whole 32 KB tiles.
// In the caller's dense layout a 400-byte pitch (w = 100) puts every odd row's segments across two sectors, which cost the
// strided passes.  Only the first pass (TMA reads) and the last pass (contiguous rows, neighbouring
// column tiles written back to back by the same CTA) touch the dense layout.  Wide matrices go through in column chunks so
// that the two intermediates stay small (and L2-friendly) whatever the width.
//   inverse:  d_in (dense) --pass--> A (tiled) --passes in place--> A = coefficients, network order, lazy range
//   forward:  A --PERM pass, per coset--> B (tiled, 2^added_bits blocks per tile) --passes in place--> last pass --> d_out (dense)
template <int F>
static int32_t lde_tiled_impl(p3gpu_ctx *ctx, const u32 *d_in, size_t h, size_t w, unsigned added_bits, u32 shift, u32 *d_out, bool *done,
                              const ShardedOut *shard = nullptr, size_t in_pitch = 0, size_t out_pitch = 0) {
    // in_pitch / out_pitch (elements, 0 = w): the matrix may be a column block of a wider row-major buffer on either side
    if (in_pitch == 0) in_pitch = w;
    if (out_pitch == 0) out_pitch = w;
    *done = false;
    const int log_n = (int)log2_floor(h);
    const int max_r = std::min(10, std::max(6, env_int("P3GPU_NTT_MAXR", 10)));
    const NetworkPlan plan = plan_passes(log_n, max_r);
    const bool enabled = pipe_mode() != 0 && env_int("P3GPU_NTT_TILED", 1);
    if (!enabled || plan.n_passes < 2 || plan.n_passes > 6) return P3GPU_OK;
    for (int k = 0; k < plan.n_passes; k++) {
        const int r = plan.bounds[k + 1] - plan.bounds[k];
        if (r < 6 || r > 10) return P3GPU_OK;
    }
    if (w % 4 != 0 || w < 8 || (reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(shard ? nullptr : d_out)) % 16 != 0) return P3GPU_OK;
    if (((in_pitch * 4) << log_n) >= (1ull << 40) || in_pitch % 4 != 0 || tensor_map_encoder() == nullptr) return P3GPU_OK;
    const size_t n_cosets = (size_t)1 << added_bits;
    // column chunk: keep B (n_cosets * h * chunk * 4 bytes) around 1 GiB, at least 64 columns
    size_t chunk = ((size_t)1 << 28) / (n_cosets * h);
    chunk = std::max<size_t>(64, chunk & ~(size_t)7);
    if (const int forced = env_int("P3GPU_NTT_CHUNK", 0)) chunk = (size_t)std::max(8, forced & ~7);   // tests: exercise the chunk loop
    const size_t w8 = (w + 7) & ~(size_t)7;
    chunk = std::min(std::min(chunk, w8), (size_t)8192);
    if (n_cosets * h * chunk * 4 > ((size_t)8 << 30)) return P3GPU_OK;   // huge blow-ups: the 64-column floor would need > 8 GiB of scratch

    const uint2 *tw_inv = nullptr, *tw = nullptr;
    P3_TRY(get_twiddles<F>(ctx, log_n, 0, Fp<F>::ONE, 1, &tw_inv));
    P3_TRY(get_twiddles<F>(ctx, log_n, (int)added_bits, shift, 0, &tw));
    void *A = nullptr, *B = nullptr;
    P3_TRY(ctx_scratch(ctx, h * chunk * 4, &A));
    P3_TRY(ctx_scratch2(ctx, n_cosets * h * chunk * 4, &B));

    // the inverse network runs its passes in reverse plan order so that its LAST pass and the forward network's FIRST pass
    // cover the same number of layers (same tile shape on the coefficient buffer)
    for (size_t col0 = 0; col0 < w; col0 += chunk) {
        const size_t wc = std::min(chunk, w - col0);
        for (int k = 0; k < plan.n_passes; k++) {          // inverse
            PassArgs a;
            memset(&a, 0, sizeof a);
            const int kk = plan.n_passes - 1 - k;            // reversed plan: bounds mirrored
            a.l0 = log_n - plan.bounds[kk + 1]; a.l1 = log_n - plan.bounds[kk];
            a.w = (u32)in_pitch; a.wc = (u32)wc; a.log_n = log_n; a.n_cosets = 1; a.in_blocks = 1;
            a.tw = tw_inv; a.tw_stride = 0;
            if (k == 0) { a.in = d_in + col0; a.in_tiled = 0; a.has_scale = 1; a.scale = inv_height_scale<F>(h); }
            else { a.in = (const u32 *)A; a.in_tiled = 1; }
            a.out = (u32 *)A; a.out_tiled = 1;
            P3_TRY(launch_pipe<F>(ctx, a));
        }
        for (int k = 0; k < plan.n_passes; k++) {          // forward, all cosets per launch
            PassArgs a;
            memset(&a, 0, sizeof a);
            a.l0 = plan.bounds[k]; a.l1 = plan.bounds[k + 1];
            a.w = (u32)out_pitch; a.wc = (u32)wc; a.log_n = log_n; a.n_cosets = (u32)n_cosets;
            a.tw = tw; a.tw_stride = h;
            if (k == 0) { a.in = (const u32 *)A; a.in_tiled = 1; a.in_blocks = 1; a.in_bitrev = 1; }
            else { a.in = (const u32 *)B; a.in_tiled = 1; a.in_blocks = (u32)n_cosets; }
            if (k == plan.n_passes - 1 && shard) {
                // the last pass stores straight into the row blocks of all ranks (peer memory): pitch = the full trace width
                a.out = nullptr; a.out_tiled = 0; a.final_reduce = 1;
                a.w = (u32)shard->w_total;
                a.shard_log_rows = (int)shard->log_rows;
                for (unsigned g = 0; g < shard->world; g++) a.shard_out[g] = shard->out[g] + shard->col_off + col0;
            }
            else if (k == plan.n_passes - 1) { a.out = d_out + col0; a.out_tiled = 0; a.out_stride = h * out_pitch; a.final_reduce = 1; }
            else { a.out = (u32 *)B; a.out_tiled = 1; }
            P3_TRY(launch_pipe<F>(ctx, a));
        }
    }
    *done = true;
    return P3GPU_OK;
}

template <int F>
static int32_t coset_lde_impl(p3gpu_ctx *ctx, const u32 *d_in, size_t h, size_t w, unsigned added_bits, u32 shift, u32 *d_out,
                              int bitrev_rows, size_t in_pitch = 0, size_t out_pitch = 0) {
    const int log_n = (int)log2_floor(h);
    const size_t n_cosets = (size_t)1 << added_bits;
    if (log_n == 0) {  // a constant polynomial: every evaluation equals the single input row
        const size_t n = n_cosets * w;
        broadcast_row<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_in, d_out, n_cosets, w);
        ctx->launches++;
        P3_CUDA(cudaGetLastError());
        return P3GPU_OK;
    }
    // the tiled pipeline unless every pass is one the cp.async kernel runs faster (pipe_mode)
    const bool pitched = (in_pitch != 0 && in_pitch != w) || (out_pitch != 0 && out_pitch != w);
    const NetworkPlan plan = plan_passes(log_n, 10);
    bool cp_async = pipe_mode() != 1;
    for (int k = 0; k < plan.n_passes; k++) cp_async = cp_async && cp_async_pass(plan.bounds[k + 1] - plan.bounds[k]);
    if (bitrev_rows && (pitched || !cp_async)) {
        bool done = false;
        P3_TRY(lde_tiled_impl<F>(ctx, d_in, h, w, added_bits, shift, d_out, &done, nullptr, in_pitch, out_pitch));
        if (done) return P3GPU_OK;
    }
    P3_CHECK((in_pitch == 0 || in_pitch == w) && (out_pitch == 0 || out_pitch == w), P3GPU_EUNSUPPORTED,
             "column-block LDE (pitch != width) needs the pipelined tiled path: bit-reversed rows, width %% 4 == 0, width >= 8, height >= 2^12");
    // 1) inverse network: evaluations on H (natural) -> coefficients in network (bit-reversed) order, scaled by 1/h
    // 2) forward networks, one per coset.  Memory block cb (h rows) holds the coset with natural index c = bitrev(cb):
    //    points shift * g_big^c * H  (radix_2_dit_parallel.rs:226-239).  The heaps of all cosets are one allocation
    //    (block cb at offset cb*h) so that the cosets run as grid.y of a single launch and share the coefficient reads in L2.
    const uint2 *tw_inv = nullptr, *tw = nullptr;
    P3_TRY(get_twiddles<F>(ctx, log_n, 0, Fp<F>::ONE, 1, &tw_inv));
    P3_TRY(get_twiddles<F>(ctx, log_n, (int)added_bits, shift, 0, &tw));
    void *coef = nullptr;
    P3_TRY(ctx_scratch(ctx, h * w * 4, &coef));
    // Two equal passes on the cp.async kernel: three launches (inverse pass 1, ntt_lde_mid_kernel, forward pass 2 of every coset)
    // instead of four, so the coefficients are written once and read once.
    const NetworkPlan run_plan = plan_passes(log_n, network_max_r());
    const int r = run_plan.bounds[1];
    if (bitrev_rows && (cp_async || pipe_mode() == 0) && run_plan.n_passes == 2 && 2 * r == log_n && r >= 7 && r <= 10 && n_cosets <= 4 &&
        lde_mid_tile_width((u32)w) != 0 && ((reinterpret_cast<uintptr_t>(d_in) | reinterpret_cast<uintptr_t>(d_out)) % 16) == 0 &&
        tensor_map_encoder() != nullptr && !env_int("P3GPU_NTT_GENERIC", 0)) {
        // inverse pass 1 runs on strided units (ntt_band_pass_kernel<..., STRIDED>) where it is eligible, else on the tile kernel;
        // both it and the fused pass store whole tiles or parts with tensor copies
        PassArgs a;
        memset(&a, 0, sizeof a);
        a.w = (u32)w; a.log_n = log_n; a.l0 = 0; a.l1 = r; a.tma_store = 1;
        a.tw = tw_inv; a.in = d_in; a.out = (u32 *)coef; a.has_scale = 1; a.scale = inv_height_scale<F>(h);
        if (band_first_pass_eligible(a)) P3_TRY(launch_band_first<F>(ctx, a));
        else P3_TRY(launch_pass<F>(ctx, a, 1, 4));
        // forward pass 2 reads and writes contiguous bands of 2^r rows: eighths of bands as single bulk copies in 8-CTA clusters
        // (ntt_band_pass_kernel; up to 48 columns ntt_band_pass_narrow_kernel) where an eighth fits a ring slot; P3GPU_NTT_BAND=0
        // keeps the tile kernel
        PassArgs b;
        memset(&b, 0, sizeof b);
        b.w = (u32)w; b.log_n = log_n; b.l0 = r; b.l1 = log_n; b.n_cosets = (u32)n_cosets;
        b.tw = tw; b.tw_stride = h; b.in = d_out; b.in_stride = h * w; b.out = d_out; b.out_stride = h * w; b.final_reduce = 1;
        const bool band = band_pass_eligible(b);
        // Tile-major plan (make_tile_major_tensor_maps): the fused pass stores each tile as one dense block of its own scratch, and
        // the 8-CTA band pass gathers each part's rows from those blocks with one tensor copy, so that the corner turn between the
        // two happens in the loads, which take short segments far better than stores do (DESIGN 4.1).  Only for whole column tiles,
        // at least two of them; P3GPU_NTT_GATHER=0 keeps the dense layout.  The scratch holds every coset: band i's output rows
        // hold tile i's blocks, which every band reads.
        const u32 ct = lde_mid_tile_width((u32)w), n_ct = (u32)w / ct;
        CUtensorMap gather_map;
        void *tiles = nullptr;
        // (The band pass's slot bounds w << r, which keeps the scratch below the 2^32 words the fused pass's offsets can address.)
        bool gather = band && w > BAND_NARROW_W && w % ct == 0 && n_ct >= 2 && n_cosets * h * w < (1ull << 32) &&
                      env_int("P3GPU_NTT_GATHER", 1) != 0;
        if (gather) {
            P3_TRY(ctx_lde_tiles(ctx, n_cosets * h * w * 4, &tiles));
            gather = make_tile_major_tensor_maps((const u32 *)tiles, ct, n_ct, r, (u32)n_cosets, (1u << r) / BAND_CL, &gather_map) == P3GPU_OK;
            if (gather) b.in = (const u32 *)tiles;
        }
        memset(&a, 0, sizeof a);
        a.w = (u32)w; a.log_n = log_n; a.l0 = r; a.l1 = log_n; a.n_cosets = (u32)n_cosets;
        a.tw = tw_inv; a.tw_stride = h; a.in = (const u32 *)coef; a.out = gather ? (u32 *)tiles : d_out; a.out_stride = h * w;
        P3_TRY(launch_lde_mid<F>(ctx, a, tw, gather));
        if (band) return launch_band<F>(ctx, b, gather ? &gather_map : nullptr);
        return launch_pass<F>(ctx, b, (unsigned)n_cosets, 4);
    }
    P3_TRY(run_network<F>(ctx, log_n, w, tw_inv, 0, 1, d_in, 0, 0, (u32 *)coef, 0, 0, 0, 0, nullptr, true, inv_height_scale<F>(h), false));
    if (bitrev_rows) {
        P3_TRY(run_network<F>(ctx, log_n, w, tw, h, (unsigned)n_cosets, (const u32 *)coef, 0, 1, d_out, h * w, 0, 0, 0, nullptr, false,
                              make_uint2(0, 0), true));
    } else {
        void *tmp = nullptr;
        P3_TRY(ctx_scratch2(ctx, h * w * 4, &tmp));
        for (size_t cb = 0; cb < n_cosets; cb++) {
            size_t c = 0;
            for (unsigned b = 0; b < added_bits; b++) c |= ((cb >> b) & 1) << (added_bits - 1 - b);
            // natural LDE row of (coset c, evaluation index j) is j * n_cosets + c
            P3_TRY(run_network<F>(ctx, log_n, w, tw + cb * h, 0, 1, (const u32 *)coef, 0, 1, d_out, 0, 1, (int)added_bits, (u32)c,
                                  (u32 *)tmp, false, make_uint2(0, 0), true));
        }
    }
    return P3GPU_OK;
}

static int32_t check_shape(int field, size_t h, size_t w, unsigned extra_bits) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "unknown field %d", field);
    P3_CHECK(w >= 1 && w < (1ull << 31), P3GPU_EINVAL, "matrix width %zu out of range", w);
    P3_CHECK(is_pow2(h), P3GPU_EINVAL, "matrix height %zu is not a power of two", h);
    const unsigned adicity = field == BABY_BEAR ? Fp<BABY_BEAR>::TWO_ADICITY : Fp<KOALA_BEAR>::TWO_ADICITY;
    P3_CHECK(log2_floor(h) + extra_bits <= adicity, P3GPU_EINVAL, "height 2^%u (+%u bits) exceeds the field's two-adicity %u",
             log2_floor(h), extra_bits, adicity);
    P3_CHECK((h << extra_bits) * w < (1ull << 40), P3GPU_EINVAL, "matrix too large");
    return P3GPU_OK;
}

int32_t ntt_dft_batch(p3gpu_ctx *ctx, int field, int kind, const u32 *d_in, u32 *d_out, size_t h, size_t w, u32 shift) {
    P3_TRY(check_shape(field, h, w, 0));
    P3_CHECK(kind >= P3GPU_DFT && kind <= P3GPU_COSET_IDFT, P3GPU_EINVAL, "unknown transform kind %d", kind);
    return field == BABY_BEAR ? dft_batch_impl<BABY_BEAR>(ctx, kind, d_in, d_out, h, w, shift)
                              : dft_batch_impl<KOALA_BEAR>(ctx, kind, d_in, d_out, h, w, shift);
}

int32_t ntt_coset_lde(p3gpu_ctx *ctx, int field, const u32 *d_in, size_t h, size_t w, unsigned added_bits, u32 shift, u32 *d_out,
                      int bitrev_rows, size_t in_pitch, size_t out_pitch) {
    P3_CHECK(added_bits <= 8, P3GPU_EINVAL, "added_bits %u too large", added_bits);
    P3_TRY(check_shape(field, h, w, added_bits));
    P3_CHECK(d_in != d_out, P3GPU_EINVAL, "coset_lde_batch cannot run in place");
    P3_CHECK((in_pitch == 0 || in_pitch >= w) && (out_pitch == 0 || out_pitch >= w), P3GPU_EINVAL, "row pitch smaller than the width");
    return field == BABY_BEAR ? coset_lde_impl<BABY_BEAR>(ctx, d_in, h, w, added_bits, shift, d_out, bitrev_rows, in_pitch, out_pitch)
                              : coset_lde_impl<KOALA_BEAR>(ctx, d_in, h, w, added_bits, shift, d_out, bitrev_rows, in_pitch, out_pitch);
}

// The LDE kept as coefficients plus one coset at a time, for traces whose whole LDE does not fit beside them.
// Coefficients: the inverse network of coset_lde_impl's generic path (network order, scaled by 1/h, lazy range) run on the trace
// itself.  Without an output remap every pass, the first one included, writes exactly the rows of its tile that it read, so the
// passes run in place and need no scratch.
template <int F>
static int32_t lde_coefficients_impl(p3gpu_ctx *ctx, u32 *d_trace, size_t h, size_t w) {
    const int log_n = (int)log2_floor(h);
    if (log_n == 0) return P3GPU_OK;   // a constant polynomial: its one coefficient is its value
    const uint2 *tw_inv = nullptr;
    P3_TRY(get_twiddles<F>(ctx, log_n, 0, Fp<F>::ONE, 1, &tw_inv));
    return run_network<F>(ctx, log_n, w, tw_inv, 0, 1, d_trace, 0, 0, d_trace, 0, 0, 0, 0, nullptr, true, inv_height_scale<F>(h), false);
}

// Memory block `coset` of the bit-reversed LDE (rows [coset h, (coset + 1) h)) from lde_coefficients_impl's coefficients: the
// forward network of that one coset with its twiddle heap, as the LDE runs it for every coset — the first pass permutes the
// coefficients (PERM pass), the last runs on the band kernel where it is eligible, as forward pass 2 of the LDE does.
template <int F>
static int32_t lde_coset_block_impl(p3gpu_ctx *ctx, const u32 *d_coef, size_t h, size_t w, unsigned added_bits, u32 shift, size_t coset,
                                    u32 *d_out) {
    const int log_n = (int)log2_floor(h);
    if (log_n == 0) {   // every evaluation of a constant is the constant
        P3_CUDA(cudaMemcpyAsync(d_out, d_coef, w * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        return P3GPU_OK;
    }
    const uint2 *tw = nullptr;
    P3_TRY(get_twiddles<F>(ctx, log_n, (int)added_bits, shift, 0, &tw));
    const uint2 *tw_c = tw + coset * h;
    const NetworkPlan plan = plan_passes(log_n, network_max_r());
    if (plan.n_passes == 2) {
        PassArgs b;
        memset(&b, 0, sizeof b);
        b.w = (u32)w; b.log_n = log_n; b.l0 = plan.bounds[1]; b.l1 = log_n; b.n_cosets = 1;
        b.tw = tw_c; b.in = d_out; b.in_stride = h * w; b.out = d_out; b.out_stride = h * w; b.final_reduce = 1;
        if (band_pass_eligible(b)) {
            PassArgs a;
            memset(&a, 0, sizeof a);
            a.w = (u32)w; a.log_n = log_n; a.l0 = 0; a.l1 = plan.bounds[1];
            a.tw = tw_c; a.in = d_coef; a.in_bitrev = 1; a.out = d_out;
            P3_TRY(launch_pass<F>(ctx, a, 1, 4));
            return launch_band<F>(ctx, b);
        }
    }
    return run_network<F>(ctx, log_n, w, tw_c, 0, 1, d_coef, 0, 1, d_out, 0, 0, 0, 0, nullptr, false, make_uint2(0, 0), true);
}

int32_t ntt_lde_coefficients(p3gpu_ctx *ctx, int field, u32 *d_trace, size_t h, size_t w) {
    P3_TRY(check_shape(field, h, w, 0));
    return field == BABY_BEAR ? lde_coefficients_impl<BABY_BEAR>(ctx, d_trace, h, w) : lde_coefficients_impl<KOALA_BEAR>(ctx, d_trace, h, w);
}

int32_t ntt_lde_coset_block(p3gpu_ctx *ctx, int field, const u32 *d_coef, size_t h, size_t w, unsigned added_bits, u32 shift, size_t coset,
                            u32 *d_out) {
    P3_CHECK(added_bits <= 8, P3GPU_EINVAL, "added_bits %u too large", added_bits);
    P3_TRY(check_shape(field, h, w, added_bits));
    P3_CHECK(coset < ((size_t)1 << added_bits), P3GPU_EINVAL, "coset %zu of an LDE with %zu cosets", coset, (size_t)1 << added_bits);
    P3_CHECK(d_coef != d_out, P3GPU_EINVAL, "the coset block cannot overwrite the coefficients");
    return field == BABY_BEAR ? lde_coset_block_impl<BABY_BEAR>(ctx, d_coef, h, w, added_bits, shift, coset, d_out)
                              : lde_coset_block_impl<KOALA_BEAR>(ctx, d_coef, h, w, added_bits, shift, coset, d_out);
}

// Column-sharded coset LDE whose result lands row-sharded on all ranks (SURVEY 8e: column blocks -> all-to-all -> row blocks).
// Column chunks a rank's block of w_local columns is exchanged in (boundaries multiples of 8 columns; P3GPU_SHARD_CHUNK, default
// 64).  Every rank computes the same list for every source rank: the chunk-major row-block layout depends on it.
std::vector<size_t> shard_chunk_bounds(size_t w_local) {
    const size_t chunk = (size_t)std::max(8, env_int("P3GPU_SHARD_CHUNK", 64) & ~7);
    const size_t n_chunks = std::max<size_t>(1, (w_local + chunk / 2) / chunk);
    std::vector<size_t> cb{0};
    for (size_t c = 1; c <= n_chunks; c++) {
        const size_t b = c == n_chunks ? w_local : (w_local * c / n_chunks) & ~(size_t)7;
        if (b > cb.back()) cb.push_back(b);
    }
    if (cb.back() != w_local) cb.push_back(w_local);
    return cb;
}

int32_t ntt_coset_lde_sharded(p3gpu_ctx *ctx, int field, const u32 *d_in, size_t h, size_t w_local, unsigned added_bits, u32 shift,
                              unsigned world, u32 *const *rank_out, size_t w_total, size_t col_off, int chunk_major) {
    P3_CHECK(added_bits <= 8, P3GPU_EINVAL, "added_bits %u too large", added_bits);
    if (w_local == 0) {   // a rank without columns (more ranks than column units) only takes part in the barriers and the hashing
        P3_TRY(check_shape(field, h, 1, added_bits));
        return P3GPU_OK;
    }
    P3_TRY(check_shape(field, h, w_local, added_bits));
    P3_CHECK(world >= 1 && world <= 16 && (world & (world - 1)) == 0, P3GPU_EINVAL, "world size %u must be a power of two <= 16", world);
    P3_CHECK(col_off + w_local <= w_total && w_total < (1ull << 31), P3GPU_EINVAL, "column block [%zu, %zu) outside the trace width %zu", col_off, col_off + w_local, w_total);
    const size_t H = h << added_bits;
    P3_CHECK(H % world == 0, P3GPU_EINVAL, "LDE height %zu not divisible by %u ranks", H, world);
    ShardedOut sh;
    memset(&sh, 0, sizeof sh);
    sh.world = world; sh.log_rows = log2_floor(H / world); sh.w_total = w_total; sh.col_off = col_off;
    // a tile of the last pass (2^r consecutive rows, r <= 10) must not straddle two ranks
    P3_CHECK(sh.log_rows >= 10 && sh.log_rows <= 31, P3GPU_EUNSUPPORTED, "sharded LDE needs at least 1024 rows per rank (have 2^%u)", sh.log_rows);
    for (unsigned g = 0; g < world; g++) { P3_CHECK(rank_out[g] != nullptr, P3GPU_EINVAL, "null output block for rank %u", g); sh.out[g] = rank_out[g]; }
    // Three ways to get the result into the row blocks (P3GPU_SHARD_MODE), compared at N = 2 on the 2^20 x 100-per-GPU LDE and on the
    // config-5 trace commit:
    //   fused  : the last pass of the transform stores every tile straight into the owner's row block: 32-byte segments over NVLink
    //            make that pass link-bound;
    //   staged : the transform runs column chunk by column chunk into a local staging buffer; as soon as a chunk is done a push kernel
    //            on a second stream copies its row blocks to their owners with 16-byte-per-lane coalesced stores while the next chunk
    //            is transformed (the push kernel shares the SMs with the persistent NTT kernel);
    //   dma    : (default) as staged, with one 2-D peer copy per destination on the copy engines instead
    //            of the push kernel.
    const char *mode = getenv("P3GPU_SHARD_MODE");
    if (!mode) mode = world == 1 ? "fused" : "dma";   // a single rank owns every row: store straight into its block, nothing to exchange
    if (chunk_major && world > 1 && strcmp(mode, "fused") == 0) mode = "dma";   // the fused stores know the row-major layout only
    if (mode && strcmp(mode, "fused") == 0 && !(chunk_major && world > 1)) {
        bool done = false;
        if (field == BABY_BEAR) P3_TRY(lde_tiled_impl<BABY_BEAR>(ctx, d_in, h, w_local, added_bits, shift, nullptr, &done, &sh));
        else P3_TRY(lde_tiled_impl<KOALA_BEAR>(ctx, d_in, h, w_local, added_bits, shift, nullptr, &done, &sh));
        P3_CHECK(done, P3GPU_EUNSUPPORTED, "sharded LDE needs the pipelined tiled path: width %% 4 == 0, width >= 8, 16-byte aligned input, 2^12 <= height");
        return P3GPU_OK;
    }
    P3_CHECK(w_local % 4 == 0 && w_total % 4 == 0 && col_off % 4 == 0, P3GPU_EUNSUPPORTED, "sharded LDE: column blocks must be multiples of 4 columns");
    if (!ctx->xchg_stream) {
        P3_CUDA(cudaStreamCreateWithFlags(&ctx->xchg_stream, cudaStreamNonBlocking));
        for (int b = 0; b < 2; b++) {
            P3_CUDA(cudaEventCreateWithFlags(&ctx->ev_stage_full[b], cudaEventDisableTiming));
            P3_CUDA(cudaEventCreateWithFlags(&ctx->ev_stage_free[b], cudaEventDisableTiming));
        }
    }
    const unsigned sh_rank_hint = (unsigned)((col_off * world) / std::max<size_t>(w_total, 1));   // ~ my rank: staggers the peers' copy order
    const std::vector<size_t> cb = shard_chunk_bounds(w_local);
    size_t wmax = 0;
    for (size_t c = 0; c + 1 < cb.size(); c++) wmax = std::max(wmax, cb[c + 1] - cb[c]);
    for (int b = 0; b < 2; b++) {
        if (ctx->stage_bytes[b] < H * wmax * 4) {
            if (ctx->stage_buf[b]) { P3_CUDA(cudaDeviceSynchronize()); P3_CUDA(cudaFree(ctx->stage_buf[b])); ctx->stage_buf[b] = nullptr; ctx->stage_bytes[b] = 0; }
            cudaError_t e = cudaMalloc(&ctx->stage_buf[b], H * wmax * 4);
            if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", H * wmax * 4, cudaGetErrorString(e)); cudaGetLastError(); return P3GPU_ENOMEM; }
            ctx->stage_bytes[b] = H * wmax * 4;
        }
    }
    for (size_t c = 0; c + 1 < cb.size(); c++) {
        const int b = (int)(c & 1);
        const size_t c0 = cb[c], wc = cb[c + 1] - c0;
        if (wc == 0) continue;
        if (c >= 2) P3_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_stage_free[b], 0));      // the push of chunk c-2 has drained this buffer
        u32 *S = (u32 *)ctx->stage_buf[b];
        if (field == BABY_BEAR) P3_TRY(coset_lde_impl<BABY_BEAR>(ctx, d_in + c0, h, wc, added_bits, shift, S, 1, w_local, wc));
        else P3_TRY(coset_lde_impl<KOALA_BEAR>(ctx, d_in + c0, h, wc, added_bits, shift, S, 1, w_local, wc));
        P3_CUDA(cudaEventRecord(ctx->ev_stage_full[b], ctx->stream));
        P3_CUDA(cudaStreamWaitEvent(ctx->xchg_stream, ctx->ev_stage_full[b], 0));
        if (mode && strcmp(mode, "dma") == 0) {
            // copy engines instead of the push kernel: one 2-D peer copy per destination rank (no SM resources, but narrow rows), each
            // on its own stream so that the copies to the different peers run concurrently; the exchange stream joins them
            const size_t R = (size_t)1 << sh.log_rows;
            for (unsigned q = 0; q < world; q++) {
                const unsigned dq = (q + sh_rank_hint) % world;            // start with a different peer on every rank
                if (!ctx->dma_stream[dq]) {
                    P3_CUDA(cudaStreamCreateWithFlags(&ctx->dma_stream[dq], cudaStreamNonBlocking));
                    P3_CUDA(cudaEventCreateWithFlags(&ctx->dma_done[dq], cudaEventDisableTiming));
                }
                P3_CUDA(cudaStreamWaitEvent(ctx->dma_stream[dq], ctx->ev_stage_full[b], 0));
                if (chunk_major)   // the chunk is one contiguous (R x wc) matrix on both sides: a plain copy at link rate
                    P3_CUDA(cudaMemcpyAsync(rank_out[dq] + R * (col_off + c0), S + (size_t)dq * R * wc, R * wc * 4, cudaMemcpyDeviceToDevice, ctx->dma_stream[dq]));
                else
                    P3_CUDA(cudaMemcpy2DAsync(rank_out[dq] + col_off + c0, w_total * 4, S + (size_t)dq * R * wc, wc * 4, wc * 4, R, cudaMemcpyDeviceToDevice,
                                              ctx->dma_stream[dq]));
                P3_CUDA(cudaEventRecord(ctx->dma_done[dq], ctx->dma_stream[dq]));
                P3_CUDA(cudaStreamWaitEvent(ctx->xchg_stream, ctx->dma_done[dq], 0));
            }
        } else {
            if (chunk_major) P3_TRY(peer_push_rows(ctx, ctx->xchg_stream, world, rank_out, S, H, wc, wc, ((size_t)1 << sh.log_rows) * (col_off + c0), sh.log_rows));
            else P3_TRY(peer_push_rows(ctx, ctx->xchg_stream, world, rank_out, S, H, wc, w_total, col_off + c0, sh.log_rows));
        }
        P3_CUDA(cudaEventRecord(ctx->ev_stage_free[b], ctx->xchg_stream));
    }
    // whatever follows on the context's stream (the barrier) comes after the last pushes
    for (int b = 0; b < 2; b++) P3_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->ev_stage_free[b], 0));
    return P3GPU_OK;
}

}  // namespace p3
