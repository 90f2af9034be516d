// Quotient of any AIR given as a constraint program (air_program.cuh): uni-stark/src/prover.rs:462-827 for the AIRs the hand-written
// Poseidon2 kernel (air.cu) does not cover.
//
// Mapping: one thread per natural index i of the quotient domain g * K.  Every thread of a warp runs the same instruction stream,
// read with uniform loads (one L1 transaction per warp and instruction), so opcodes never diverge.  Slots live in shared memory laid
// out [slot][thread] (128 threads per block): conflict-free, and the footprint — slots x 512 B + constraints x 16 B for the
// alpha-power table — is known at compile time of the program, so `create` can refuse a program that does not fit before anything
// launches.  Trace values are read straight from the committed bit-reversed LDE (memory row bitrev(i), next row bitrev(i + 2^q)).
#include "common.h"
#include "air_program.cuh"

struct p3gpu_air_program {
    int device = 0;
    p3::AirProgram prog;
    p3::AirInsn *d_insns = nullptr;
};

namespace p3 {

struct AirQArgs {
    const AirInsn *prog;
    u32 n_insns, n_cons;
    const u32 *lde;
    size_t width;
    const uint4 *apow;          // alpha^(K - 1 - k), k < K
    const u32 *zh, *izh;        // Z_H and 1 / Z_H by i mod 2^q
    const u32 *pubs;
    u32 *q;
    AirDomain d;
};

template <int F> struct AirDevEnv {
    const AirQArgs *a;
    const uint4 *ap;
    u32 *sl;                    // this thread's slot 0; slot s at sl[s * AIR_BLOCK]
    const u32 *row, *nrow;
    __device__ __forceinline__ AirInsn insn(u32 pc) const {
        const uint2 v = __ldg(reinterpret_cast<const uint2 *>(a->prog) + pc);
        return AirInsn{v.x, v.y};
    }
    __device__ __forceinline__ u32 &slot(u32 s) { return sl[s * AIR_BLOCK]; }
    __device__ __forceinline__ void set_rows(u32 m, u32 mn) { row = a->lde + (size_t)m * a->width; nrow = a->lde + (size_t)mn * a->width; }
    __device__ __forceinline__ u32 local(u32 c) const { return __ldg(row + c); }
    __device__ __forceinline__ u32 next(u32 c) const { return __ldg(nrow + c); }
    __device__ __forceinline__ u32 pub(u32 k) const { return __ldg(a->pubs + k); }
    __device__ __forceinline__ uint4 apow(u32 k) const { return ap[k]; }
    __device__ __forceinline__ u32 zh(u32 i) const { return __ldg(a->zh + (i & ((1u << a->d.q) - 1u))); }
    __device__ __forceinline__ u32 inv_zh(u32 i) const { return __ldg(a->izh + (i & ((1u << a->d.q) - 1u))); }
};

template <int F> __global__ void __launch_bounds__(AIR_BLOCK) air_program_quotient_kernel(const AirQArgs a) {
    extern __shared__ uint4 air_sm[];
    for (u32 t = threadIdx.x; t < a.n_cons; t += AIR_BLOCK) air_sm[t] = __ldg(a.apow + t);
    __syncthreads();
    const u32 i = blockIdx.x * AIR_BLOCK + threadIdx.x;
    if (i >= (1u << a.d.log_q)) return;
    AirDevEnv<F> env;
    env.a = &a;
    env.ap = air_sm;
    env.sl = reinterpret_cast<u32 *>(air_sm + a.n_cons) + threadIdx.x;
    reinterpret_cast<uint4 *>(a.q)[i] = air_row_quotient<F>(env, a.d, a.n_insns, i);
}

int32_t air_program_create(p3gpu_ctx *ctx, int field, const p3gpu_air_node *nodes, size_t n_nodes, const u32 *constraints, size_t n_constraints,
                           u32 width, u32 n_public, p3gpu_air_program **out) {
    std::string err;
    AirProgram prog;
    const int32_t rc = air_compile(field, nodes, n_nodes, constraints, n_constraints, width, n_public, prog, err);
    P3_CHECK(rc == P3GPU_OK, rc, "%s", err.c_str());
    std::unique_ptr<p3gpu_air_program> p(new p3gpu_air_program);
    p->device = ctx->device;
    P3_CUDA(cudaMalloc(&p->d_insns, std::max<size_t>(prog.insns.size(), 1) * sizeof(AirInsn)));
    if (!prog.insns.empty())
        P3_CUDA(cudaMemcpy(p->d_insns, prog.insns.data(), prog.insns.size() * sizeof(AirInsn), cudaMemcpyHostToDevice));
    p->prog = std::move(prog);
    *out = p.release();
    return P3GPU_OK;
}

void air_program_destroy(p3gpu_air_program *prog) {
    if (!prog) return;
    int cur = 0;
    if (cudaGetDevice(&cur) == cudaSuccess && cudaSetDevice(prog->device) == cudaSuccess) {
        cudaFree(prog->d_insns);
        cudaSetDevice(cur);
    }
    delete prog;
}

int32_t air_program_info(const p3gpu_air_program *prog, size_t *n_insns, size_t *n_slots, size_t *n_cons) {
    P3_CHECK(prog != nullptr, P3GPU_EINVAL, "null program");
    if (n_insns) *n_insns = prog->prog.insns.size();
    if (n_slots) *n_slots = prog->prog.n_slots;
    if (n_cons) *n_cons = prog->prog.n_constraints;
    return P3GPU_OK;
}

template <int F>
static int32_t air_quotient_launch(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *d_lde, unsigned log_q, unsigned log_n,
                                   const u32 *pubs, const u32 *alpha, u32 *d_q) {
    const AirProgram &p = pg->prog;
    for (u32 k = 0; k < p.n_public; k++) P3_CHECK(pubs[k] < Fp<F>::P, P3GPU_EINVAL, "public value %u is not a canonical Montgomery word", k);
    for (int d = 0; d < 4; d++) P3_CHECK(alpha[d] < Fp<F>::P, P3GPU_EINVAL, "alpha is not a canonical Montgomery element");
    std::vector<u32> zh, izh;
    AirQArgs qa;
    qa.d = air_domain<F>(log_q, log_n, p.uses, zh, izh);
    const std::vector<uint4> ap = air_alpha_table<F>(alpha, p.n_constraints);
    // one staging copy: alpha table | Z_H | 1/Z_H | public values
    const size_t nz = zh.size(), words = (size_t)p.n_constraints * 4 + 2 * nz + p.n_public;
    std::vector<u32> host(std::max<size_t>(words, 1));
    if (!ap.empty()) memcpy(host.data(), ap.data(), ap.size() * 16);
    u32 *h = host.data() + (size_t)p.n_constraints * 4;
    std::copy(zh.begin(), zh.end(), h);
    std::copy(izh.begin(), izh.end(), h + nz);
    std::copy(pubs, pubs + p.n_public, h + 2 * nz);
    void *tab = nullptr;
    P3_TRY(ctx_scratch2(ctx, host.size() * 4, &tab));
    P3_CUDA(cudaMemcpyAsync(tab, host.data(), host.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    u32 *dt = static_cast<u32 *>(tab);
    qa.prog = pg->d_insns; qa.n_insns = (u32)p.insns.size(); qa.n_cons = p.n_constraints;
    qa.lde = d_lde; qa.width = p.width;
    qa.apow = reinterpret_cast<const uint4 *>(dt);
    qa.zh = dt + (size_t)p.n_constraints * 4; qa.izh = qa.zh + nz; qa.pubs = qa.izh + nz;
    qa.q = d_q;
    const size_t smem = air_smem_bytes(p.n_slots, p.n_constraints);
    auto kern = air_program_quotient_kernel<F>;
    if (smem > 48 * 1024) P3_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const size_t n = (size_t)1 << log_q;
    kern<<<(unsigned)((n + AIR_BLOCK - 1) / AIR_BLOCK), AIR_BLOCK, smem, ctx->stream>>>(qa);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t air_program_quotient(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *d_lde, unsigned log_lde, unsigned log_q, unsigned log_n,
                             const u32 *pubs, const u32 *alpha, u32 *d_q) {
    P3_CHECK(pg->device == ctx->device, P3GPU_EINVAL, "AIR program was created on device %d, the context is on device %d", pg->device, ctx->device);
    const int field = pg->prog.field;
    const unsigned two_adicity = field == BABY_BEAR ? Fp<BABY_BEAR>::TWO_ADICITY : Fp<KOALA_BEAR>::TWO_ADICITY;
    P3_CHECK(log_n <= log_q && log_q <= log_lde && log_lde <= two_adicity, P3GPU_EINVAL,
             "need log_trace_height %u <= log_quotient_size %u <= log_lde_height %u <= %u", log_n, log_q, log_lde, two_adicity);
    P3_CHECK(log_q - log_n <= AIR_MAX_RATE_BITS, P3GPU_EUNSUPPORTED, "quotient domain 2^%u over a trace of 2^%u rows: at most %u extra bits",
             log_q, log_n, AIR_MAX_RATE_BITS);
    P3_CHECK(pg->prog.n_public == 0 || pubs != nullptr, P3GPU_EINVAL, "the program reads %u public values, none given", pg->prog.n_public);
    P3_CHECK(reinterpret_cast<uintptr_t>(d_q) % 16 == 0 && reinterpret_cast<uintptr_t>(d_lde) % 4 == 0, P3GPU_EINVAL, "quotient: misaligned buffer");
    P3_CHECK(air_smem_bytes(pg->prog.n_slots, pg->prog.n_constraints) <= 227 * 1024, P3GPU_EUNSUPPORTED, "AIR program needs more shared memory than a block has");
    if (field == BABY_BEAR) return air_quotient_launch<BABY_BEAR>(ctx, pg, d_lde, log_q, log_n, pubs, alpha, d_q);
    return air_quotient_launch<KOALA_BEAR>(ctx, pg, d_lde, log_q, log_n, pubs, alpha, d_q);
}

}  // namespace p3
