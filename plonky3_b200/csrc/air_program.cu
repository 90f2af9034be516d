// Quotient of any AIR given as a constraint program (air_program.cuh): uni-stark/src/prover.rs:462-827 for the AIRs the hand-written
// Poseidon2 kernel (air.cu) does not cover.
//
// Mapping: one thread per natural index i of the quotient domain g * K.  Every thread of a warp runs the same instruction stream,
// read with uniform loads (one L1 transaction per warp and instruction), so opcodes never diverge.  Slots live in shared memory laid
// out [slot][thread] (128 threads per block): conflict-free, and the footprint — slots x 512 B + constraints x 16 B for the
// alpha-power table — is known at compile time of the program, so `create` can refuse a program that does not fit before anything
// launches.  Trace values are read straight from the committed bit-reversed LDE (memory row bitrev(i), next row bitrev(i + 2^q)),
// preprocessed values the same way from the committed preprocessed LDE, periodic values from row i mod (p_max * 2^q) of the small
// periodic table (read-only path; at most p_max * 2^q x n_periodic words, cache-resident).  A program that reads neither runs the
// instance without them (EXT = false): the same code as before they existed.
#include "common.h"
#include "air_program.cuh"

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
    const u32 *pre;             // preprocessed LDE (EXT instances only)
    size_t pre_width;
    const u32 *periodic;        // periodic table, row-major (EXT instances only)
    u32 n_periodic;
    AirDomain d;
};

template <int F> struct AirDevEnv {
    const AirQArgs *a;
    const uint4 *ap;
    u32 *sl;                    // this thread's slot 0; slot s at sl[s * AIR_BLOCK]
    const u32 *row, *nrow, *prow, *pnrow, *per;
    __device__ __forceinline__ AirInsn insn(u32 pc) const {
        const uint2 v = __ldg(reinterpret_cast<const uint2 *>(a->prog) + pc);
        return AirInsn{v.x, v.y};
    }
    __device__ __forceinline__ u32 &slot(u32 s) { return sl[s * AIR_BLOCK]; }
    __device__ __forceinline__ void set_rows(u32 m, u32 mn) { row = a->lde + (size_t)m * a->width; nrow = a->lde + (size_t)mn * a->width; }
    __device__ __forceinline__ void set_ext_rows(u32 m, u32 mn, u32 pr) {
        prow = a->pre + (size_t)m * a->pre_width; pnrow = a->pre + (size_t)mn * a->pre_width; per = a->periodic + (size_t)pr * a->n_periodic;
    }
    __device__ __forceinline__ u32 local(u32 c) const { return __ldg(row + c); }
    __device__ __forceinline__ u32 pre_local(u32 c) const { return __ldg(prow + c); }
    __device__ __forceinline__ u32 pre_next(u32 c) const { return __ldg(pnrow + c); }
    __device__ __forceinline__ u32 periodic(u32 k) const { return __ldg(per + k); }
    __device__ __forceinline__ u32 next(u32 c) const { return __ldg(nrow + c); }
    __device__ __forceinline__ u32 pub(u32 k) const { return __ldg(a->pubs + k); }
    __device__ __forceinline__ uint4 apow(u32 k) const { return ap[k]; }
    __device__ __forceinline__ u32 zh(u32 i) const { return __ldg(a->zh + (i & ((1u << a->d.q) - 1u))); }
    __device__ __forceinline__ u32 inv_zh(u32 i) const { return __ldg(a->izh + (i & ((1u << a->d.q) - 1u))); }
};

template <int F, bool EXT> __global__ void __launch_bounds__(AIR_BLOCK) air_program_quotient_kernel(const AirQArgs a) {
    extern __shared__ uint4 air_sm[];
    for (u32 t = threadIdx.x; t < a.n_cons; t += AIR_BLOCK) air_sm[t] = __ldg(a.apow + t);
    __syncthreads();
    const u32 i = blockIdx.x * AIR_BLOCK + threadIdx.x;
    if (i >= (1u << a.d.log_q)) return;
    AirDevEnv<F> env;
    env.a = &a;
    env.ap = air_sm;
    env.sl = reinterpret_cast<u32 *>(air_sm + a.n_cons) + threadIdx.x;
    reinterpret_cast<uint4 *>(a.q)[i] = air_row_quotient<F, EXT>(env, a.d, a.n_insns, i);
}

// Row-sharded instance (p3gpu_air_quotient_sharded_dev): one rank's row block of the row-sharded commit, whose quotient domain is
// the LDE domain.  One thread per block row m: natural index i = bitrev(row0 + m), the same air_row_quotient as the dense kernel,
// its value stored at q[m] (the block's bit-reversed slice).  Local columns are read in place from the rank's chunk-major block,
// next-row columns from the chunk-major block of the one rank holding every next row of this block (air_shard_next_rank), at
// local row bitrev(i + 2^q) mod R; both through the unit table (AirShardRow), which sits in shared memory behind the slots.
// Periodic values as in the dense kernel (every rank holds the whole small table).  A program without AIR_USES_NEXT never reads
// the peer's block.  The peer's rows are final before this kernel runs, because the sharded commit ends in a barrier, and stay
// unchanged until every rank is done with them, because a row block is written only by the commit and the exchange after the
// quotient (ShardedTrace.quotient_values) starts with a barrier.
struct AirShardQArgs {
    AirQArgs q;                 // the dense arguments: program, tables, output; q.lde / q.width unused
    const u32 *own, *peer;      // my row block; the row block holding my points' next rows (my own when the program reads none)
    const u64 *units;           // n_units entries, one per 8 columns (air_shard_units)
    u32 n_units, n_slots, row0, rows;
    unsigned log_rows;
};

template <int F> struct AirShardDevEnv : AirDevEnv<F> {
    const AirShardQArgs *s;
    const u64 *tab;             // the unit table in shared memory
    AirShardRow cur, nxt;
    __device__ __forceinline__ void set_rows(u32 m, u32 mn) {
        cur = AirShardRow{s->own, tab, air_shard_locate(m, s->log_rows).row};
        nxt = AirShardRow{s->peer, tab, air_shard_locate(mn, s->log_rows).row};
    }
    __device__ __forceinline__ void set_ext_rows(u32, u32, u32 pr) { this->per = this->a->periodic + (size_t)pr * this->a->n_periodic; }
    __device__ __forceinline__ u32 local(u32 c) const { return cur.ld(c); }
    __device__ __forceinline__ u32 next(u32 c) const { return nxt.ld(c); }
    // the sharded entry refuses a program with preprocessed columns
    __device__ __forceinline__ u32 pre_local(u32) const { return 0u; }
    __device__ __forceinline__ u32 pre_next(u32) const { return 0u; }
};

template <int F, bool EXT> __global__ void __launch_bounds__(AIR_BLOCK) air_program_quotient_sharded_kernel(const AirShardQArgs a) {
    extern __shared__ uint4 air_sm[];
    for (u32 t = threadIdx.x; t < a.q.n_cons; t += AIR_BLOCK) air_sm[t] = __ldg(a.q.apow + t);
    u64 *tab = reinterpret_cast<u64 *>(reinterpret_cast<u32 *>(air_sm + a.q.n_cons) + (size_t)a.n_slots * AIR_BLOCK);
    for (u32 t = threadIdx.x; t < a.n_units; t += AIR_BLOCK) tab[t] = __ldg(a.units + t);
    __syncthreads();
    const u32 m = blockIdx.x * AIR_BLOCK + threadIdx.x;
    if (m >= a.rows) return;
    AirShardDevEnv<F> env;
    env.a = &a.q;
    env.ap = air_sm;
    env.sl = reinterpret_cast<u32 *>(air_sm + a.q.n_cons) + threadIdx.x;
    env.s = &a;
    env.tab = tab;
    reinterpret_cast<uint4 *>(a.q.q)[m] = air_row_quotient<F, EXT>(env, a.q.d, a.q.n_insns, air_bitrev(a.row0 + m, a.q.d.log_q));
}

int32_t air_program_create(p3gpu_ctx *ctx, int field, const p3gpu_air_node *nodes, size_t n_nodes, const u32 *constraints, size_t n_constraints,
                           const p3gpu_air_layout &layout, p3gpu_air_program **out, bool check) {
    std::string err;
    AirProgram prog;
    const int32_t rc = air_compile(field, nodes, n_nodes, constraints, n_constraints, layout.width, layout.n_public, layout.preprocessed_width,
                                   layout.n_periodic, prog, err, check ? AIR_CHECK_LIMITS : AIR_QUOTIENT_LIMITS);
    P3_CHECK(rc == P3GPU_OK, rc, "%s", err.c_str());
    std::unique_ptr<p3gpu_air_program> p(new p3gpu_air_program);
    p->device = ctx->device;
    p->check = check;
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

// The launch arguments of either instance: checks the public values and alpha, builds the domain and stages the tables in one
// copy: alpha table | Z_H | 1/Z_H | public values | (8-byte aligned) `units`, the sharded instance's unit table (*d_units).
template <int F>
static int32_t air_quotient_args(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *d_lde, const u32 *d_pre, const u32 *d_periodic,
                                 unsigned log_periodic_rows, unsigned log_q, unsigned log_n, const u32 *pubs, const u32 *alpha, u32 *d_q,
                                 const std::vector<u64> &units, AirQArgs &qa, const u64 **d_units) {
    const AirProgram &p = pg->prog;
    for (u32 k = 0; k < p.n_public; k++) P3_CHECK(pubs[k] < Fp<F>::P, P3GPU_EINVAL, "public value %u is not a canonical Montgomery word", k);
    for (int d = 0; d < 4; d++) P3_CHECK(alpha[d] < Fp<F>::P, P3GPU_EINVAL, "alpha is not a canonical Montgomery element");
    std::vector<u32> zh, izh;
    qa.d = air_domain<F>(log_q, log_n, p.uses, zh, izh);
    qa.d.periodic_mask = (1u << log_periodic_rows) - 1u;
    const std::vector<uint4> ap = air_alpha_table<F>(alpha, p.n_constraints);
    const size_t nz = zh.size(), words = (size_t)p.n_constraints * 4 + 2 * nz + p.n_public;
    const size_t unit_at = (words + 1) & ~(size_t)1;
    std::vector<u32> host(std::max<size_t>(units.empty() ? words : unit_at + 2 * units.size(), 1));
    if (!ap.empty()) memcpy(host.data(), ap.data(), ap.size() * 16);
    u32 *h = host.data() + (size_t)p.n_constraints * 4;
    std::copy(zh.begin(), zh.end(), h);
    std::copy(izh.begin(), izh.end(), h + nz);
    std::copy(pubs, pubs + p.n_public, h + 2 * nz);
    if (!units.empty()) memcpy(host.data() + unit_at, units.data(), units.size() * 8);
    void *tab = nullptr;
    P3_TRY(ctx_scratch2(ctx, host.size() * 4, &tab));
    P3_CUDA(cudaMemcpyAsync(tab, host.data(), host.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    u32 *dt = static_cast<u32 *>(tab);
    qa.prog = pg->d_insns; qa.n_insns = (u32)p.insns.size(); qa.n_cons = p.n_constraints;
    qa.lde = d_lde; qa.width = p.width;
    qa.apow = reinterpret_cast<const uint4 *>(dt);
    qa.zh = dt + (size_t)p.n_constraints * 4; qa.izh = qa.zh + nz; qa.pubs = qa.izh + nz;
    qa.q = d_q;
    qa.pre = d_pre; qa.pre_width = p.pre_width;
    qa.periodic = d_periodic; qa.n_periodic = p.n_periodic;
    if (d_units) *d_units = reinterpret_cast<const u64 *>(dt + unit_at);
    return P3GPU_OK;
}

template <int F>
static int32_t air_quotient_launch(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *d_lde, const u32 *d_pre, const u32 *d_periodic,
                                   unsigned log_periodic_rows, unsigned log_q, unsigned log_n, const u32 *pubs, const u32 *alpha, u32 *d_q) {
    const AirProgram &p = pg->prog;
    AirQArgs qa;
    P3_TRY(air_quotient_args<F>(ctx, pg, d_lde, d_pre, d_periodic, log_periodic_rows, log_q, log_n, pubs, alpha, d_q, {}, qa, nullptr));
    const size_t smem = air_smem_bytes(p.n_slots, p.n_constraints);
    auto kern = (p.uses & AIR_USES_EXT) ? air_program_quotient_kernel<F, true> : air_program_quotient_kernel<F, false>;
    if (smem > 48 * 1024) P3_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const size_t n = (size_t)1 << log_q;
    kern<<<(unsigned)((n + AIR_BLOCK - 1) / AIR_BLOCK), AIR_BLOCK, smem, ctx->stream>>>(qa);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t air_program_quotient(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *d_lde, unsigned log_lde, const u32 *d_pre, unsigned log_pre,
                             const u32 *d_periodic, unsigned log_periodic_rows, unsigned log_q, unsigned log_n, const u32 *pubs,
                             const u32 *alpha, u32 *d_q, bool layout_entry) {
    P3_CHECK(pg->device == ctx->device, P3GPU_EINVAL, "AIR program was created on device %d, the context is on device %d", pg->device, ctx->device);
    P3_CHECK(!pg->check, P3GPU_EINVAL,
             "the AIR program was created with p3gpu_air_check_program_create: evaluate the quotient of a p3gpu_air_program_create program");
    const AirProgram &p = pg->prog;
    const int field = p.field;
    P3_CHECK(layout_entry || (p.pre_width == 0 && p.n_periodic == 0), P3GPU_EINVAL,
             "the AIR program has preprocessed or periodic columns: evaluate it with p3gpu_air_quotient_layout_dev");
    const unsigned two_adicity = field == BABY_BEAR ? Fp<BABY_BEAR>::TWO_ADICITY : Fp<KOALA_BEAR>::TWO_ADICITY;
    P3_CHECK(log_n <= log_q && log_q <= log_lde && log_lde <= two_adicity, P3GPU_EINVAL,
             "need log_trace_height %u <= log_quotient_size %u <= log_lde_height %u <= %u", log_n, log_q, log_lde, two_adicity);
    P3_CHECK(log_q - log_n <= AIR_MAX_RATE_BITS, P3GPU_EUNSUPPORTED, "quotient domain 2^%u over a trace of 2^%u rows: at most %u extra bits",
             log_q, log_n, AIR_MAX_RATE_BITS);
    P3_CHECK(pg->prog.n_public == 0 || pubs != nullptr, P3GPU_EINVAL, "the program reads %u public values, none given", pg->prog.n_public);
    P3_CHECK(reinterpret_cast<uintptr_t>(d_q) % 16 == 0 && reinterpret_cast<uintptr_t>(d_lde) % 4 == 0, P3GPU_EINVAL, "quotient: misaligned buffer");
    P3_CHECK(air_smem_bytes(pg->prog.n_slots, pg->prog.n_constraints) <= 227 * 1024, P3GPU_EUNSUPPORTED, "AIR program needs more shared memory than a block has");
    // preprocessed LDE: given iff the layout has preprocessed columns, read like the trace LDE's quotient-domain prefix
    P3_CHECK((p.pre_width > 0) == (d_pre != nullptr), P3GPU_EINVAL, "preprocessed LDE %s, the program's preprocessed width is %u",
             d_pre ? "given" : "missing", p.pre_width);
    if (d_pre) {
        P3_CHECK(log_q <= log_pre && log_pre <= two_adicity, P3GPU_EINVAL, "preprocessed LDE of 2^%u rows: need 2^%u <= height <= 2^%u", log_pre,
                 log_q, two_adicity);
        P3_CHECK(reinterpret_cast<uintptr_t>(d_pre) % 4 == 0, P3GPU_EINVAL, "quotient: misaligned preprocessed LDE");
    }
    // periodic table: given iff the layout has periodic columns, at most one row per quotient point
    P3_CHECK((p.n_periodic > 0) == (d_periodic != nullptr), P3GPU_EINVAL, "periodic table %s, the program has %u periodic columns",
             d_periodic ? "given" : "missing", p.n_periodic);
    if (d_periodic) {
        P3_CHECK(log_periodic_rows <= log_q, P3GPU_EINVAL, "periodic table of 2^%u rows over a quotient domain of 2^%u", log_periodic_rows, log_q);
        P3_CHECK(reinterpret_cast<uintptr_t>(d_periodic) % 4 == 0, P3GPU_EINVAL, "quotient: misaligned periodic table");
    } else {
        log_periodic_rows = 0;
    }
    if (field == BABY_BEAR)
        return air_quotient_launch<BABY_BEAR>(ctx, pg, d_lde, d_pre, d_periodic, log_periodic_rows, log_q, log_n, pubs, alpha, d_q);
    return air_quotient_launch<KOALA_BEAR>(ctx, pg, d_lde, d_pre, d_periodic, log_periodic_rows, log_q, log_n, pubs, alpha, d_q);
}

template <int F>
static int32_t air_quotient_sharded_launch(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *own, const u32 *peer, const std::vector<u64> &units,
                                           size_t smem, u32 row0, unsigned log_rows, const u32 *d_periodic, unsigned log_periodic_rows,
                                           unsigned log_lde, unsigned log_n, const u32 *pubs, const u32 *alpha, u32 *d_q) {
    const AirProgram &p = pg->prog;
    AirShardQArgs sa;
    P3_TRY(air_quotient_args<F>(ctx, pg, nullptr, nullptr, d_periodic, log_periodic_rows, log_lde, log_n, pubs, alpha, d_q, units, sa.q, &sa.units));
    sa.own = own; sa.peer = peer;
    sa.n_units = (u32)units.size(); sa.n_slots = p.n_slots; sa.row0 = row0; sa.rows = 1u << log_rows; sa.log_rows = log_rows;
    auto kern = (p.uses & AIR_USES_EXT) ? air_program_quotient_sharded_kernel<F, true> : air_program_quotient_sharded_kernel<F, false>;
    if (smem > 48 * 1024) P3_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<sa.rows / AIR_BLOCK, AIR_BLOCK, smem, ctx->stream>>>(sa);
    ctx->launches++;
    P3_CUDA(cudaGetLastError());
    return P3GPU_OK;
}

int32_t air_program_quotient_sharded(p3gpu_ctx *ctx, const p3gpu_air_program *pg, unsigned world, unsigned rank, u32 *const *rows,
                                     const size_t *col_starts, const u32 *d_periodic, unsigned log_periodic_rows, unsigned log_lde, unsigned log_n,
                                     const u32 *pubs, const u32 *alpha, u32 *d_q) {
    P3_CHECK(pg->device == ctx->device, P3GPU_EINVAL, "AIR program was created on device %d, the context is on device %d", pg->device, ctx->device);
    P3_CHECK(!pg->check, P3GPU_EINVAL,
             "the AIR program was created with p3gpu_air_check_program_create: evaluate the quotient of a p3gpu_air_program_create program");
    const AirProgram &p = pg->prog;
    const int field = p.field;
    P3_CHECK(p.pre_width == 0, P3GPU_EUNSUPPORTED, "sharded AIR quotient: the program has %u preprocessed columns (no sharded preprocessed trace)",
             p.pre_width);
    const unsigned two_adicity = field == BABY_BEAR ? Fp<BABY_BEAR>::TWO_ADICITY : Fp<KOALA_BEAR>::TWO_ADICITY;
    P3_CHECK(log_n <= log_lde && log_lde <= two_adicity, P3GPU_EINVAL, "sharded AIR quotient: need log_trace_height %u <= log_lde_height %u <= %u",
             log_n, log_lde, two_adicity);
    // the quotient domain is the LDE domain: its 2^log_lde points are the LDE's rows, and rank g owns points bitrev(g R + m)
    P3_CHECK(log_lde - log_n <= AIR_MAX_RATE_BITS, P3GPU_EUNSUPPORTED,
             "sharded AIR quotient: the quotient domain is the LDE domain, 2^%u over a trace of 2^%u rows: at most %u extra bits", log_lde, log_n,
             AIR_MAX_RATE_BITS);
    const unsigned log_g = log2_floor(world);
    P3_CHECK(log_lde >= log_g && log_lde - log_g >= 10, P3GPU_EUNSUPPORTED,
             "sharded AIR quotient: 2^%u LDE rows over %u ranks (at least 1024 rows per rank, as the sharded commit)", log_lde, world);
    const unsigned log_rows = log_lde - log_g;
    P3_CHECK(p.n_public == 0 || pubs != nullptr, P3GPU_EINVAL, "the program reads %u public values, none given", p.n_public);
    P3_CHECK(reinterpret_cast<uintptr_t>(d_q) % 16 == 0, P3GPU_EINVAL, "sharded AIR quotient: misaligned quotient slice");
    for (unsigned g = 0; g < world; g++)
        P3_CHECK(reinterpret_cast<uintptr_t>(rows[g]) % 4 == 0, P3GPU_EINVAL, "sharded AIR quotient: misaligned row block of rank %u", g);
    P3_CHECK((p.n_periodic > 0) == (d_periodic != nullptr), P3GPU_EINVAL, "periodic table %s, the program has %u periodic columns",
             d_periodic ? "given" : "missing", p.n_periodic);
    if (d_periodic) {
        P3_CHECK(log_periodic_rows <= log_lde, P3GPU_EINVAL, "periodic table of 2^%u rows over a quotient domain of 2^%u", log_periodic_rows, log_lde);
        P3_CHECK(reinterpret_cast<uintptr_t>(d_periodic) % 4 == 0, P3GPU_EINVAL, "sharded AIR quotient: misaligned periodic table");
    } else {
        log_periodic_rows = 0;
    }
    std::vector<u64> units;
    P3_TRY(air_shard_units(world, col_starts, (size_t)1 << log_rows, p.width, units));
    const size_t base = air_smem_bytes(p.n_slots, p.n_constraints), smem = base + units.size() * 8;
    P3_CHECK(smem <= 227 * 1024, P3GPU_EUNSUPPORTED,
             "sharded AIR quotient needs %zu bytes of shared memory, a block has %d: %u slots x %u B + %u constraints x 16 B + %zu units x 8 B",
             smem, 227 * 1024, p.n_slots, AIR_BLOCK * 4, p.n_constraints, units.size());
    const u32 *peer = (p.uses & AIR_USES_NEXT) ? rows[air_shard_next_rank(rank, log_g, log_lde - log_n)] : rows[rank];
    const u32 row0 = rank << log_rows;
    if (field == BABY_BEAR)
        return air_quotient_sharded_launch<BABY_BEAR>(ctx, pg, rows[rank], peer, units, smem, row0, log_rows, d_periodic, log_periodic_rows, log_lde,
                                                      log_n, pubs, alpha, d_q);
    return air_quotient_sharded_launch<KOALA_BEAR>(ctx, pg, rows[rank], peer, units, smem, row0, log_rows, d_periodic, log_periodic_rows, log_lde,
                                                   log_n, pubs, alpha, d_q);
}

// ---- hand-written AIR quotient kernels (keccak_air.cu, blake3_air.cu, poseidon1_air.cu) -----------------------------------
template <int F>
static int32_t hand_quotient_launch(p3gpu_ctx *ctx, const void *kern, u32 n_constraints, unsigned warps, size_t smem, u32 uses, const u32 *d_lde,
                                    unsigned log_n, const u32 *alpha, u32 *d_q, const u32 *consts, unsigned lanes, const AirHandShard *shard) {
    for (int d = 0; d < 4; d++) P3_CHECK(alpha[d] < Fp<F>::P, P3GPU_EINVAL, "alpha is not a canonical Montgomery element");
    AirHandQArgs qa;
    std::vector<u32> zh, izh;
    qa.d = air_domain<F>(log_n + 1, log_n, uses, zh, izh);
    for (int j = 0; j < 2; j++) { qa.zh[j] = zh[j]; qa.izh[j] = izh[j]; }
    const std::vector<uint4> ap = air_alpha_table<F>(alpha, n_constraints);
    std::vector<u64> units;
    qa.units = nullptr; qa.n_units = 0; qa.row0 = 0; qa.rows = 0;
    size_t points = (size_t)1 << qa.d.log_q;
    if (shard) {
        points = points / shard->world;
        P3_TRY(air_shard_units(shard->world, shard->col_starts, points, shard->width, units));
        qa.n_units = (u32)units.size(); qa.row0 = (u32)(shard->rank * points); qa.rows = (u32)points;
        smem += units.size() * 8;
    }
    void *tab = nullptr;
    P3_TRY(ctx_scratch2(ctx, ap.size() * 16 + units.size() * 8, &tab));
    P3_CUDA(cudaMemcpyAsync(tab, ap.data(), ap.size() * 16, cudaMemcpyHostToDevice, ctx->stream));
    if (shard) {                                                     // the unit table behind the alpha table (16-byte entries)
        qa.units = reinterpret_cast<const u64 *>(static_cast<uint4 *>(tab) + ap.size());
        P3_CUDA(cudaMemcpyAsync(const_cast<u64 *>(qa.units), units.data(), units.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    }
    qa.lde = d_lde; qa.apow = static_cast<const uint4 *>(tab); qa.q = d_q;
    qa.consts = consts; qa.lanes = lanes;
    P3_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // `lanes` lanes per point, persistent blocks
    const size_t per_block = (size_t)warps * 32 / lanes;
    const unsigned grid = (unsigned)std::min<size_t>((size_t)ctx->sm_count, (points + per_block - 1) / per_block);
    void *args[] = {&qa};
    P3_CUDA(cudaLaunchKernel(kern, dim3(grid), dim3(32 * warps), args, smem, ctx->stream));
    ctx->launches++;
    return P3GPU_OK;
}

int32_t air_hand_quotient(p3gpu_ctx *ctx, int field, const char *name, const void *kern_babybear, const void *kern_koalabear, u32 n_constraints,
                          unsigned warps, size_t smem, u32 uses, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q,
                          const u32 *consts, unsigned lanes, const AirHandShard *shard) {
    P3_CHECK(field == BABY_BEAR || field == KOALA_BEAR, P3GPU_EUNSUPPORTED, "%s AIR: unsupported field %d", name, field);
    const unsigned two_adicity = field == BABY_BEAR ? Fp<BABY_BEAR>::TWO_ADICITY : Fp<KOALA_BEAR>::TWO_ADICITY;
    P3_CHECK(log_n + 1 <= log_lde && log_lde <= two_adicity, P3GPU_EINVAL,
             "%s AIR quotient: need log_trace_height %u + 1 <= log_lde_height %u <= %u", name, log_n, log_lde, two_adicity);
    P3_CHECK(reinterpret_cast<uintptr_t>(d_lde) % 4 == 0 && reinterpret_cast<uintptr_t>(d_q) % 4 == 0, P3GPU_EINVAL,
             "%s AIR quotient: misaligned buffer", name);
    if (shard) {
        // the quotient domain must be the LDE domain: then the 2N points are the 2N LDE rows, and rank g owns points bitrev(g R + m)
        P3_CHECK(log_lde == log_n + 1, P3GPU_EINVAL, "%s AIR sharded quotient: the LDE must have 2N rows (log_blowup 1), not 2^%u over 2^%u", name,
                 log_lde, log_n);
        P3_CHECK(shard->world >= 1 && shard->world <= 16 && (shard->world & (shard->world - 1)) == 0 && shard->rank < shard->world, P3GPU_EINVAL,
                 "%s AIR sharded quotient: world %u must be a power of two <= 16, rank %u below it", name, shard->world, shard->rank);
        P3_CHECK(((size_t)2 << log_n) / shard->world >= 1024, P3GPU_EUNSUPPORTED,
                 "%s AIR sharded quotient: %zu rows per rank (at least 1024, as the sharded commit)", name, ((size_t)2 << log_n) / shard->world);
    }
    if (field == BABY_BEAR)
        return hand_quotient_launch<BABY_BEAR>(ctx, kern_babybear, n_constraints, warps, smem, uses, d_lde, log_n, alpha, d_q, consts, lanes, shard);
    return hand_quotient_launch<KOALA_BEAR>(ctx, kern_koalabear, n_constraints, warps, smem, uses, d_lde, log_n, alpha, d_q, consts, lanes, shard);
}

int32_t air_shard_units(unsigned world, const size_t *col_starts, size_t rows, size_t width, std::vector<u64> &units) {
    P3_CHECK(col_starts[world] == width, P3GPU_EINVAL, "the column blocks cover %zu columns, the trace has %zu", col_starts[world], width);
    P3_CHECK(width < (1u << 16) && rows * width < (1ull << 48), P3GPU_EUNSUPPORTED, "row block of %zu x %zu: too large for the unit table", rows,
             width);
    std::vector<size_t> segs;
    P3_TRY(shard_col_segments(world, col_starts, rows, segs));
    units.assign((width + AIR_UNIT - 1) / AIR_UNIT, 0);
    for (size_t s = 0; s < segs.size(); s += 3) {
        const size_t c0 = segs[s], c1 = segs[s + 1], off = segs[s + 2];
        P3_CHECK(c0 % AIR_UNIT == 0 && (c1 % AIR_UNIT == 0 || c1 == width), P3GPU_EINVAL,
                 "column segment [%zu, %zu) does not start and end on a multiple of %u columns", c0, c1, AIR_UNIT);
        for (size_t u = c0 / AIR_UNIT; u * AIR_UNIT < c1; u++) units[u] = air_unit_entry(off - c0, c1 - c0);
    }
    return P3GPU_OK;
}

int32_t air_check_window(const char *name, size_t col0, size_t col1, size_t width) {
    P3_CHECK(col0 <= col1 && col1 <= width, P3GPU_EINVAL, "%s AIR: column window [%zu, %zu) outside the trace width %zu", name, col0, col1, width);
    return P3GPU_OK;
}

}  // namespace p3
