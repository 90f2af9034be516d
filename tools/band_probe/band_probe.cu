// Probe for the coset LDE's band pass (ntt_band_pass_kernel): the three numbers its design rests on, measured on the device.
//   1. in-place streaming of the forward pass 2 buffer (2^21 x 100 u32 = 839 MB read + 839 MB written) as 100 KB 1-D bulk
//      copies, persistent 4-CTA clusters, a 2-deep ring per CTA (the load of chunk k+1 waits until the store of chunk k-1 has
//      left its buffer);
//   2. the DSMEM rate of the radix-4 exchange in 4-CTA clusters: each CTA reads 3/4 of its 100 KB quarter's worth from its peers
//      and writes 3/4 back, between two cluster barriers, 64 times (the bands a CTA takes at 2^20 x 100, blowup 2);
//   3. cudaOccupancyMaxActiveClusters for clusters of 4 and 8 CTAs at 221 KB of dynamic shared memory, 512 threads;
//   4. the first pass's strided units (2^20 x 100: unit L = rows L + 1024 i, i < 1024), 15 clusters of 8 CTAs, a 3-slot ring, no
//      arithmetic: CTA q moves rows i in [128q, 128q + 128) of each unit from one 419 MB buffer to another, either as ONE 3-D tensor
//      copy in and ONE 3-D tensor store out per part, or as 128 1-D bulk copies of 400 bytes each way (4 per lane of one warp).
//   5. the fused middle pass's traffic at 2^20 x 100, two cosets, no arithmetic: 132 persistent CTAs with one lane each load row
//      tile T (coefficient rows T * 1024 + rho) through the inverse-layout 5-D box and store it once per coset through the
//      forward-layout box (rows L + 1024 i, T = bitrev10(L)), 419 MB read + 839 MB written, in two shapes:
//      (a) 20-column tiles, 2 buffers, tile k + 2 loaded once tile k's last store has been read out (ntt_lde_mid_kernel);
//      (b) 8-column tiles (one 4-column tile per row tile), a 5-stage ring, 3 tiles held at once, each stage released once its
//          tile's two stores have been read out; each CTA takes whole row tiles;
//      and each shape once with its loads only and once with its stores only (each stage loaded once, then stored from repeatedly).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 band_probe.cu -o band_probe
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <vector>
typedef unsigned u32;
constexpr int THREADS = 512;
constexpr u32 W = 100, QROWS = 256, QWORDS = QROWS * W, QBYTES = QWORDS * 4;   // one quarter band: 256 rows x 100 columns
constexpr size_t SMEM = 2 * (QBYTES + 1024 * 8) + 64;                          // 2 x (quarter + its twiddles) + barriers

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } } while (0)

__device__ __forceinline__ u32 sa(const void *p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(u32 bar, u32 parity) {
    asm volatile("{ .reg .pred p; WAIT_%=: mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1; @!p bra WAIT_%=; }" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned; barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__global__ void __launch_bounds__(THREADS, 1) stream_kernel(u32 *buf, u32 n_chunks) {
    extern __shared__ __align__(128) unsigned char smem[];
    u32 *data = reinterpret_cast<u32 *>(smem);
    unsigned long long *full = reinterpret_cast<unsigned long long *>(smem + SMEM - 64);
    if (threadIdx.x != 0) return;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sa(full)));
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sa(full + 1)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    auto load = [&](u32 c, u32 b) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa(full + b)), "r"(QBYTES) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(sa(data + b * (QWORDS + 2048))), "l"(buf + (size_t)c * QWORDS), "r"(QBYTES), "r"(sa(full + b)) : "memory");
    };
    u32 c = blockIdx.x, k = 0;
    if (c < n_chunks) load(c, 0);
    for (; c < n_chunks; c += gridDim.x, k++) {
        const u32 b = k & 1;
        if (c + gridDim.x < n_chunks) {
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the store of chunk k-1 has left buffer b^1
            load(c + gridDim.x, b ^ 1);
        }
        mbar_wait(sa(full + b), (k >> 1) & 1);
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     ::"l"(buf + (size_t)c * QWORDS), "r"(sa(data + b * (QWORDS + 2048))), "r"(QBYTES) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// rows j, j + 256, j + 512, j + 768 of a band are row j of the cluster's four quarters; CTA q takes rows [64q, 64q + 64)
__global__ void __launch_bounds__(THREADS, 1) dsmem_kernel(u32 iters, u32 *sink) {
    extern __shared__ __align__(128) unsigned char smem[];
    u32 *data = reinterpret_cast<u32 *>(smem);
    for (u32 i = threadIdx.x; i < QWORDS; i += THREADS) data[i] = i;
    u32 q;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(q));
    u32 peer[4];
    for (u32 p = 0; p < 4; p++) asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer[p]) : "r"(sa(data)), "r"(p));
    u32 acc = 0;
    cluster_sync();
    for (u32 it = 0; it < iters; it++) {
        for (u32 i = threadIdx.x; i < (QROWS / 4) * W; i += THREADS) {
            const u32 off = (q * (QROWS / 4) * W + i) * 4;
            u32 x[4];
#pragma unroll
            for (int p = 0; p < 4; p++) asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(x[p]) : "r"(peer[p] + off) : "memory");
            const u32 t0 = x[0] + x[2], t1 = x[1] + x[3], t2 = x[0] ^ x[2], t3 = x[1] ^ x[3];
            x[0] = t0 + t1; x[1] = t0 ^ t1; x[2] = t2 + t3; x[3] = t2 ^ t3;
#pragma unroll
            for (int p = 0; p < 4; p++) asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(peer[p] + off), "r"(x[p]) : "memory");
        }
        cluster_sync();
        acc += data[(threadIdx.x * 37u + it) % QWORDS];
        cluster_sync();
    }
    if (acc == 0x9e3779b9u) sink[0] = acc;
}

// 4. strided units: 2^SU_LOG units of 2^SU_LOG rows (row L + 2^SU_LOG * i), SU_RQ rows of each per CTA, 3-slot ring per CTA
constexpr int SU_LOG = 10;
constexpr u32 SU_CL = 8, SU_RQ = (1u << SU_LOG) / SU_CL, SU_PWORDS = SU_RQ * W, SU_PBYTES = SU_PWORDS * 4;
constexpr size_t SU_SMEM = 3 * (size_t)SU_PBYTES + 8192 + 64;   // as the band pass's ring: 3 parts + twiddles + barriers

template <bool TENSOR>
__global__ void __launch_bounds__(32, 1) strided_kernel(const __grid_constant__ CUtensorMap imap, const __grid_constant__ CUtensorMap omap,
                                                        const u32 *src, u32 *dst) {
    extern __shared__ __align__(128) unsigned char smem[];
    u32 *data = reinterpret_cast<u32 *>(smem);
    unsigned long long *full = reinterpret_cast<unsigned long long *>(smem + SU_SMEM - 64);
    u32 q;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(q));
    const u32 n_clusters = gridDim.x / SU_CL, cid = blockIdx.x / SU_CL, lane = threadIdx.x;
    const u32 n = ((1u << SU_LOG) - 1 - cid) / n_clusters + 1;
    if (lane == 0) {
        for (int s = 0; s < 3; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sa(full + s)), "r"(TENSOR ? 1 : 32));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();
    auto load = [&](u32 k) {
        const u32 s = k % 3, L = cid + k * n_clusters;
        u32 *part = data + s * SU_PWORDS;
        if (TENSOR) {
            if (lane != 0) return;
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa(full + s)), "r"(SU_PBYTES) : "memory");
            asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                         ::"r"(sa(part)), "l"(reinterpret_cast<unsigned long long>(&imap)), "r"(0), "r"(L), "r"(q * SU_RQ), "r"(sa(full + s)) : "memory");
        } else {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa(full + s)), "r"(SU_PBYTES / 32) : "memory");
            for (u32 j = lane; j < SU_RQ; j += 32)
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(sa(part + j * W)), "l"(src + ((size_t)L + ((size_t)(q * SU_RQ + j) << SU_LOG)) * W), "r"(W * 4), "r"(sa(full + s)) : "memory");
        }
    };
    auto store = [&](u32 k) {
        const u32 s = k % 3, L = cid + k * n_clusters;
        const u32 *part = data + s * SU_PWORDS;
        if (TENSOR) {
            if (lane != 0) return;
            asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                         ::"l"(reinterpret_cast<unsigned long long>(&omap)), "r"(sa(part)), "r"(0), "r"(L), "r"(q * SU_RQ) : "memory");
        } else {
            for (u32 j = lane; j < SU_RQ; j += 32)
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                             ::"l"(dst + ((size_t)L + ((size_t)(q * SU_RQ + j) << SU_LOG)) * W), "r"(sa(part + j * W)), "r"(W * 4) : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    };
    for (u32 k = 0; k < 3 && k < n; k++) load(k);
    for (u32 k = 0; k < n; k++) {
        mbar_wait(sa(full + k % 3), (k / 3) & 1);
        cluster_sync();   // the band pass's one cluster barrier per period
        store(k);
        if (k + 3 < n) {
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // this lane's stores have read slot k % 3 out
            __syncwarp();
            load(k + 3);
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    cluster_sync();
}

typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                             const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
// (column, unit L, i) over a 2^(2 SU_LOG) x W matrix: row L + 2^SU_LOG * i; box (W, 1, SU_RQ) = one part, dense in shared memory
static int unit_map(EncodeFn enc, void *base, CUtensorMap *tm) {
    cuuint64_t dims[3] = {W, 1ull << SU_LOG, 1ull << SU_LOG}, strides[2] = {(cuuint64_t)W * 4, ((cuuint64_t)W * 4) << SU_LOG};
    cuuint32_t box[3] = {W, 1, SU_RQ}, es[3] = {1, 1, 1};
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("cuTensorMapEncodeTiled: %d\n", (int)r); return 1; }
    return 0;
}

// 5. the fused middle pass's loads and stores; BW-column tiles, NS stages, HELD tiles waiting for their stores at once
constexpr u32 MP_LOG = 10, MP_R = 1u << MP_LOG, MP_E = 32, MP_COSETS = 2;   // r = 10: E1 = E2 = 32
template <u32 BW> __host__ __device__ constexpr u32 mp_box_bytes() { return MP_E * (MP_E + 1) * BW * 4; }   // 32 groups of 32 rows + a zero pad row
template <u32 BW, u32 NS> constexpr size_t mp_smem() { return NS * (size_t)mp_box_bytes<BW>() + 64; }

// LOADS / STORES = false: that side's copies are left out (without loads, each stage is loaded once and stored from repeatedly)
template <u32 BW, u32 NS, u32 HELD, bool WHOLE_ROWS, bool LOADS = true, bool STORES = true>
__global__ void __launch_bounds__(32, 1) mid_kernel(const __grid_constant__ CUtensorMap imap, const __grid_constant__ CUtensorMap omap) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned long long *full = reinterpret_cast<unsigned long long *>(smem + NS * (size_t)mp_box_bytes<BW>());
    if (threadIdx.x != 0) return;
    constexpr u32 NCT = (W + BW - 1) / BW;
    const u32 n = WHOLE_ROWS ? ((MP_R - 1 - blockIdx.x) / gridDim.x + 1) * NCT : (MP_R * NCT - 1 - blockIdx.x) / gridDim.x + 1;
    auto tile = [&](u32 k, u32 &col, u32 &L) {
        const u32 t = WHOLE_ROWS ? (blockIdx.x + (k / NCT) * gridDim.x) * NCT + k % NCT : blockIdx.x + k * gridDim.x;
        col = (t % NCT) * BW; L = t / NCT;
    };
    for (u32 s = 0; s < NS; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sa(full + s)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    auto load = [&](u32 k) {
        u32 col, L;
        tile(k, col, L);
        const u32 s = k % NS, T = __brev(L) >> (32 - MP_LOG);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sa(full + s)), "r"(mp_box_bytes<BW>()) : "memory");
        asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
                     ::"r"(sa(smem + s * (size_t)mp_box_bytes<BW>())), "l"(reinterpret_cast<unsigned long long>(&imap)), "r"(col), "r"(0), "r"(0),
                       "r"(0), "r"(T), "r"(sa(full + s)) : "memory");
    };
    for (u32 k = 0; k < NS && k < n; k++) load(k);
    for (u32 k = 0; k < n; k++) {
        u32 col, L;
        tile(k, col, L);
        const u32 s = k % NS;
        if (LOADS || k < NS) mbar_wait(sa(full + s), (k / NS) & 1);
        for (u32 cs = 0; cs < MP_COSETS && STORES; cs++) {
            asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                         ::"l"(reinterpret_cast<unsigned long long>(&omap)), "r"(sa(smem + s * (size_t)mp_box_bytes<BW>())), "r"(col), "r"(0), "r"(0),
                           "r"(L), "r"(cs) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            if (HELD == 1) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the next coset rewrites the buffer
        }
        // the stores of tile k + 1 - HELD have been read out: its stage takes tile k + 1 - HELD + NS
        asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(MP_COSETS * (HELD - 1)) : "memory");
        if (LOADS && k + 1 >= HELD && k + 1 - HELD + NS < n) load(k + 1 - HELD + NS);
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// the fused pass's maps (make_pass_tensor_map at r = 10): inverse layout (column, row in group, group, 0, T) over 2^20 x W, groups of
// 32 rows (rho = group * 32 + row); forward layout (column, row in group, group, L, coset) over MP_COSETS blocks, row L + 1024 rho
static int mid_map(EncodeFn enc, void *base, bool fwd, u32 bw, CUtensorMap *tm) {
    const cuuint64_t p = (cuuint64_t)W * 4;
    cuuint64_t dims[5] = {W, MP_E, MP_E, fwd ? MP_R : 1, fwd ? MP_COSETS : MP_R};
    cuuint64_t strides[4] = {fwd ? p << MP_LOG : p, fwd ? p << (MP_LOG + 5) : p << 5, p, fwd ? p << (2 * MP_LOG) : p << MP_LOG};
    cuuint32_t box[5] = {bw, MP_E + 1, MP_E, 1, 1}, es[5] = {1, 1, 1, 1, 1};
    const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 5, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { printf("cuTensorMapEncodeTiled: %d\n", (int)r); return 1; }
    return 0;
}

template <u32 BW, u32 NS, u32 HELD, bool WHOLE_ROWS, bool LOADS = true, bool STORES = true>
static int run_mid(EncodeFn enc, u32 *coef, u32 *out, int sms, const char *what) {
    CUtensorMap imap, omap;
    if (mid_map(enc, coef, false, BW, &imap) || mid_map(enc, out, true, BW, &omap)) return 1;
    constexpr size_t smem = mp_smem<BW, NS>();
    auto kern = mid_kernel<BW, NS, HELD, WHOLE_ROWS, LOADS, STORES>;
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    std::vector<float> ts;
    for (int rep = 0; rep < 22; rep++) {
        CK(cudaEventRecord(e0));
        kern<<<sms, 32, smem>>>(imap, omap);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep >= 2) ts.push_back(ms);
    }
    std::sort(ts.begin(), ts.end());
    const double bytes = ((LOADS ? 1.0 : 0.0) + (STORES ? MP_COSETS : 0)) * ((size_t)W * 4 << (2 * MP_LOG));
    printf("fused middle pass traffic 2^%u x %u, %u cosets, %s: %zu B boxes, %u stages, %u held, %d CTAs: median of %zu %.3f ms (min %.3f, max %.3f) = %.0f GB/s\n",
           2 * MP_LOG, W, MP_COSETS, what, (size_t)mp_box_bytes<BW>(), NS, HELD, sms, ts.size(), ts[ts.size() / 2], ts[0], ts.back(),
           bytes / (ts[ts.size() / 2] * 1e-3) / 1e9);
    return 0;
}

template <typename K, typename... A>
static cudaError_t launch_cluster(K kern, u32 grid, u32 cl, A... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(THREADS); cfg.dynamicSmemBytes = SMEM;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cl; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}

static int active_clusters(const void *kern, u32 cl, int *out) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(cl * 64); cfg.blockDim = dim3(THREADS); cfg.dynamicSmemBytes = SMEM;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = cl; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
    cfg.attrs = &attr; cfg.numAttrs = 1;
    CK(cudaOccupancyMaxActiveClusters(out, kern, &cfg));
    return 0;
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device: %s, %d SMs, smem/block optin %zu\n", prop.name, prop.multiProcessorCount, prop.sharedMemPerBlockOptin);
    CK(cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
    CK(cudaFuncSetAttribute(dsmem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM));
    // 3. occupancy
    int nc4 = 0, nc8 = 0;
    if (active_clusters((const void *)stream_kernel, 4, &nc4) || active_clusters((const void *)stream_kernel, 8, &nc8)) return 1;
    printf("dynamic smem %zu B, %d threads: max active clusters: size 4 -> %d (%d SMs), size 8 -> %d (%d SMs)\n", SMEM, THREADS, nc4, 4 * nc4,
           nc8, 8 * nc8);
    if (nc4 == 0) return 1;
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    // 1. streaming
    const u32 n_chunks = (2u << 20) / QROWS;   // 2^21 rows of 100 columns = 8192 quarter bands
    const size_t bytes = (size_t)n_chunks * QBYTES;
    u32 *buf;
    CK(cudaMalloc(&buf, bytes));
    CK(cudaMemset(buf, 1, bytes));
    for (u32 cl : {4u, 8u}) {
        const u32 grid = cl * (cl == 4 ? nc4 : nc8);
        if (grid == 0) continue;
        std::vector<float> ts;
        for (int rep = 0; rep < 12; rep++) {
            CK(cudaEventRecord(e0));
            CK(launch_cluster(stream_kernel, grid, cl, buf, n_chunks));
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rep >= 2) ts.push_back(ms);
        }
        std::sort(ts.begin(), ts.end());
        printf("stream in place, cluster %u, %u CTAs: %zu MB read + written: median %.3f ms (min %.3f, max %.3f) = %.0f GB/s\n", cl, grid,
               bytes >> 20, ts[ts.size() / 2], ts[0], ts.back(), 2.0 * bytes / (ts[ts.size() / 2] * 1e-3) / 1e9);
    }
    // 2. DSMEM exchange
    u32 *sink;
    CK(cudaMalloc(&sink, 4));
    const u32 iters = 64, grid = 4 * nc4;
    std::vector<float> ts;
    for (int rep = 0; rep < 12; rep++) {
        CK(cudaEventRecord(e0));
        CK(launch_cluster(dsmem_kernel, grid, 4, iters, sink));
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (rep >= 2) ts.push_back(ms);
    }
    std::sort(ts.begin(), ts.end());
    const double remote = 2.0 * 0.75 * QBYTES * iters * grid;   // bytes crossing between SMs (reads + writes)
    printf("dsmem radix-4 exchange, %u CTAs x %u bands: median %.3f ms (min %.3f, max %.3f) = %.1f us per band, %.0f GB/s between SMs\n", grid,
           iters, ts[ts.size() / 2], ts[0], ts.back(), ts[ts.size() / 2] * 1e3 / iters, remote / (ts[ts.size() / 2] * 1e-3) / 1e9);
    CK(cudaFree(buf)); CK(cudaFree(sink));
    // 4. strided units, buffer to buffer
    EncodeFn enc = nullptr;
    cudaDriverEntryPointQueryResult qres;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", (void **)&enc, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || enc == nullptr) { printf("no cuTensorMapEncodeTiled\n"); return 1; }
    const size_t sbytes = ((size_t)W * 4) << (2 * SU_LOG);
    u32 *src, *dst;
    CK(cudaMalloc(&src, sbytes)); CK(cudaMalloc(&dst, sbytes));
    CK(cudaMemset(src, 1, sbytes)); CK(cudaMemset(dst, 0, sbytes));
    CUtensorMap imap, omap;
    if (unit_map(enc, src, &imap) || unit_map(enc, dst, &omap)) return 1;
    for (int tensor = 1; tensor >= 0; tensor--) {
        const void *kern = tensor ? (const void *)strided_kernel<true> : (const void *)strided_kernel<false>;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SU_SMEM));
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(15 * SU_CL); cfg.blockDim = dim3(32); cfg.dynamicSmemBytes = SU_SMEM;
        cudaLaunchAttribute attr;
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = SU_CL; attr.val.clusterDim.y = 1; attr.val.clusterDim.z = 1;
        cfg.attrs = &attr; cfg.numAttrs = 1;
        std::vector<float> st;
        for (int rep = 0; rep < 22; rep++) {
            CK(cudaEventRecord(e0));
            if (tensor) CK(cudaLaunchKernelEx(&cfg, strided_kernel<true>, imap, omap, (const u32 *)src, dst));
            else CK(cudaLaunchKernelEx(&cfg, strided_kernel<false>, imap, omap, (const u32 *)src, dst));
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
            if (rep >= 2) st.push_back(ms);
        }
        std::vector<u32> chk(4096);
        CK(cudaMemcpy(chk.data(), dst + sbytes / 4 - chk.size(), chk.size() * 4, cudaMemcpyDeviceToHost));
        const bool copied = std::all_of(chk.begin(), chk.end(), [](u32 v) { return v == 0x01010101u; });
        CK(cudaMemset(dst, 0, sbytes));
        std::sort(st.begin(), st.end());
        printf("strided units 2^%d x %u, 15 x %u CTAs, %s: %zu MB read + %zu MB written: median %.3f ms (min %.3f, max %.3f) = %.0f GB/s%s\n",
               2 * SU_LOG, W, SU_CL, tensor ? "3-D tensor copies" : "1-D row copies", sbytes >> 20, sbytes >> 20, st[st.size() / 2], st[0],
               st.back(), 2.0 * sbytes / (st[st.size() / 2] * 1e-3) / 1e9, copied ? "" : " (COPY WRONG)");
    }
    CK(cudaFree(src)); CK(cudaFree(dst));
    // 5. the fused middle pass's traffic
    u32 *coef, *out;
    CK(cudaMalloc(&coef, sbytes)); CK(cudaMalloc(&out, MP_COSETS * sbytes));
    CK(cudaMemset(coef, 1, sbytes)); CK(cudaMemset(out, 0, MP_COSETS * sbytes));
    if (run_mid<20, 2, 1, false>(enc, coef, out, prop.multiProcessorCount, "(a) 20-column tiles, 2 buffers") ||
        run_mid<8, 5, 3, true>(enc, coef, out, prop.multiProcessorCount, "(b) 8-column tiles, 5-stage ring, whole row tiles per CTA") ||
        run_mid<20, 2, 1, false, true, false>(enc, coef, out, prop.multiProcessorCount, "(a) loads only") ||
        run_mid<20, 2, 1, false, false, true>(enc, coef, out, prop.multiProcessorCount, "(a) stores only") ||
        run_mid<8, 5, 3, true, true, false>(enc, coef, out, prop.multiProcessorCount, "(b) loads only") ||
        run_mid<8, 5, 3, true, false, true>(enc, coef, out, prop.multiProcessorCount, "(b) stores only"))
        return 1;
    CK(cudaFree(coef)); CK(cudaFree(out));
    return 0;
}
