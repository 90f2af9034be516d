// Constraint programs: an AIR given as a symbolic expression DAG (the reference's SymbolicExpression, air/src/symbolic/expression.rs),
// compiled once into a register program that air_program.cu's quotient kernel interprets over the quotient domain and
// air_check.cu's check kernel interprets over the trace domain.
//
// This header holds everything that is not a CUDA launch — the node validation, the compiler, the per-instruction semantics, the
// per-row quotient evaluation and the per-row constraint check — so host C++ can include it (tests/cpp/air_program_check.cpp and,
// for the EXT instance, tests/cpp/air_layout_check.cpp run the quotient against the oracle on the CPU, tests/cpp/air_shard_check.cpp
// the row-sharded quotient over chunk-major row blocks, tests/cpp/air_check_host.cpp the check) exactly as the kernels do.
//
//   nodes        p3gpu_air_node {op, a, b, imm} in topological order (operands refer only to earlier nodes)
//   compile      drop dead nodes; per constraint in assertion order emit its not yet emitted cone (post-order), then FOLD it;
//                slots by liveness (an operand's slot is released at its last use, before the result is allocated), so the slot
//                count is the maximum number of simultaneously live values
//   instruction  2 words: op_dst = op | dst << 4, arg = operand (binary: a | b << 16; leaf: column / public index / Montgomery
//                constant; FOLD: dst is the constraint index, arg the slot).  Node ops 0-10 are their own opcodes; the preprocessed
//                and periodic leaves (node ops 16-18) become opcodes 12-14, so every opcode fits the 4-bit field
//   fold         acc += c_k * alpha^(K - 1 - k) (the first constraint gets the highest power, air/src/symbolic/builder.rs:482-511),
//                lazily in 64 bits per coefficient; quotient = acc / Z_H(x)
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/p3gpu.h"
#include "field.cuh"

namespace p3 {

constexpr u32 AIR_OP_FOLD = 11;                 // instruction-only op, after the node ops P3GPU_AIR_CONST .. P3GPU_AIR_MUL
constexpr u32 AIR_OP_PRE_LOCAL = 12, AIR_OP_PRE_NEXT = 13, AIR_OP_PERIODIC = 14;     // P3GPU_AIR_PREPROCESSED_LOCAL / _NEXT, PERIODIC
constexpr u32 AIR_MAX_SLOTS = 384;              // 384 slots x 128 threads x 4 B = 192 KiB of shared memory per block
constexpr u32 AIR_MAX_CONSTRAINTS = 2048;       // alpha-power table: 32 KiB of shared memory
// A check program (air_check.cu) has no alpha table and keeps its slots in global memory: its limits are the instruction fields'
// (16-bit slot operands, 28-bit FOLD constraint index).
constexpr u32 AIR_CHECK_MAX_SLOTS = 65535, AIR_CHECK_MAX_CONSTRAINTS = (1u << 28) - 1;
struct AirLimits { u32 max_slots, max_constraints; };
constexpr AirLimits AIR_QUOTIENT_LIMITS = {AIR_MAX_SLOTS, AIR_MAX_CONSTRAINTS}, AIR_CHECK_LIMITS = {AIR_CHECK_MAX_SLOTS, AIR_CHECK_MAX_CONSTRAINTS};
constexpr u32 AIR_BLOCK = 128;
constexpr unsigned AIR_MAX_RATE_BITS = 8;       // q = log_quotient_size - log_trace_height <= 8: Z_H tables of <= 256 entries

// uses_mask bits
constexpr u32 AIR_USES_NEXT = 1, AIR_USES_SELECTORS = 2, AIR_USES_PUBLIC = 4;
constexpr u32 AIR_USES_PRE_LOCAL = 8, AIR_USES_PRE_NEXT = 16, AIR_USES_PERIODIC = 32;
constexpr u32 AIR_USES_EXT = AIR_USES_PRE_LOCAL | AIR_USES_PRE_NEXT | AIR_USES_PERIODIC;

struct AirInsn { u32 op_dst, arg; };

struct AirProgram {
    int field = 0;
    u32 width = 0, n_public = 0, pre_width = 0, n_periodic = 0;
    u32 n_slots = 0, n_constraints = 0, uses = 0;
    std::vector<AirInsn> insns;
};

}  // namespace p3

// A compiled program on the device: a quotient program (p3gpu_air_program_create*) or a check program
// (p3gpu_air_check_program_create), which only the check entry points run.
struct p3gpu_air_program {
    int device = 0;
    bool check = false;
    p3::AirProgram prog;
    p3::AirInsn *d_insns = nullptr;
};

namespace p3 {

inline size_t air_smem_bytes(u32 n_slots, u32 n_constraints) { return (size_t)n_constraints * 16 + (size_t)n_slots * AIR_BLOCK * 4; }

// Validates the node list and compiles it.  Returns P3GPU_OK, P3GPU_EINVAL (malformed nodes / constraints) or P3GPU_EUNSUPPORTED
// (beyond the slot or constraint limit of `lim`); `err` says why.
// pre_width / n_periodic: the preprocessed columns and periodic columns the leaves may read (0: none).
inline int32_t air_compile(int field, const p3gpu_air_node *nodes, size_t n_nodes, const uint32_t *constraints, size_t n_constraints,
                           u32 width, u32 n_public, u32 pre_width, u32 n_periodic, AirProgram &out, std::string &err,
                           const AirLimits &lim = AIR_QUOTIENT_LIMITS) {
    auto fail = [&](int32_t code, const std::string &m) { err = m; return code; };
    if (field != BABY_BEAR && field != KOALA_BEAR) return fail(P3GPU_EUNSUPPORTED, "AIR program: unsupported field " + std::to_string(field));
    const u32 P = field == BABY_BEAR ? Fp<BABY_BEAR>::P : Fp<KOALA_BEAR>::P;
    if (n_nodes > 0 && nodes == nullptr) return fail(P3GPU_EINVAL, "AIR program: null node list");
    if (n_constraints > 0 && constraints == nullptr) return fail(P3GPU_EINVAL, "AIR program: null constraint list");
    if (n_nodes >= (1ull << 31)) return fail(P3GPU_EINVAL, "AIR program: too many nodes");
    for (size_t i = 0; i < n_nodes; i++) {
        const p3gpu_air_node &n = nodes[i];
        const std::string at = "AIR program: node " + std::to_string(i) + ": ";
        switch (n.op) {
            case P3GPU_AIR_CONST:
                if (n.imm >= P) return fail(P3GPU_EINVAL, at + "constant is not a canonical Montgomery word");
                break;
            case P3GPU_AIR_MAIN_LOCAL: case P3GPU_AIR_MAIN_NEXT:
                if (n.a >= width) return fail(P3GPU_EINVAL, at + "column " + std::to_string(n.a) + " >= width " + std::to_string(width));
                break;
            case P3GPU_AIR_PUBLIC:
                if (n.a >= n_public) return fail(P3GPU_EINVAL, at + "public value " + std::to_string(n.a) + " >= " + std::to_string(n_public));
                break;
            case P3GPU_AIR_IS_FIRST_ROW: case P3GPU_AIR_IS_LAST_ROW: case P3GPU_AIR_IS_TRANSITION:
                break;
            case P3GPU_AIR_PREPROCESSED_LOCAL: case P3GPU_AIR_PREPROCESSED_NEXT:
                if (n.a >= pre_width)
                    return fail(P3GPU_EINVAL, at + "preprocessed column " + std::to_string(n.a) + " >= preprocessed width " + std::to_string(pre_width));
                break;
            case P3GPU_AIR_PERIODIC:
                if (n.a >= n_periodic)
                    return fail(P3GPU_EINVAL, at + "periodic column " + std::to_string(n.a) + " >= " + std::to_string(n_periodic));
                break;
            case P3GPU_AIR_ADD: case P3GPU_AIR_SUB: case P3GPU_AIR_MUL:
                if (n.b >= i) return fail(P3GPU_EINVAL, at + "operand b = " + std::to_string(n.b) + " is not an earlier node");
                // fallthrough
            case P3GPU_AIR_NEG:
                if (n.a >= i) return fail(P3GPU_EINVAL, at + "operand a = " + std::to_string(n.a) + " is not an earlier node");
                break;
            default:
                return fail(P3GPU_EINVAL, at + "unknown op " + std::to_string(n.op));
        }
    }
    for (size_t k = 0; k < n_constraints; k++)
        if (constraints[k] >= n_nodes) return fail(P3GPU_EINVAL, "AIR program: constraint " + std::to_string(k) + " names node " +
                                                               std::to_string(constraints[k]) + " of " + std::to_string(n_nodes));
    if (n_constraints > lim.max_constraints)
        return fail(P3GPU_EUNSUPPORTED, "AIR program: " + std::to_string(n_constraints) + " constraints (at most " + std::to_string(lim.max_constraints) + ")");

    auto is_binary = [](u32 op) { return op == P3GPU_AIR_ADD || op == P3GPU_AIR_SUB || op == P3GPU_AIR_MUL; };
    // schedule: events are node indices (compute) or ~k (fold constraint k)
    std::vector<int64_t> events;
    std::vector<uint8_t> state(n_nodes, 0);     // 0 new, 1 on the stack, 2 emitted
    std::vector<std::pair<u32, int>> stack;
    for (size_t k = 0; k < n_constraints; k++) {
        if (state[constraints[k]] != 2) {
            stack.push_back({constraints[k], 0});
            while (!stack.empty()) {
                auto &top = stack.back();
                const p3gpu_air_node &n = nodes[top.first];
                const int n_ops = is_binary(n.op) ? 2 : n.op == P3GPU_AIR_NEG ? 1 : 0;
                if (top.second < n_ops) {
                    const u32 c = top.second == 0 ? n.a : n.b;
                    top.second++;
                    if (state[c] == 0) { state[c] = 1; stack.push_back({c, 0}); }
                } else {
                    state[top.first] = 2;
                    events.push_back(top.first);
                    stack.pop_back();
                }
            }
        }
        events.push_back(~(int64_t)k);
    }
    // liveness: last event that reads each node
    std::vector<size_t> last(n_nodes, 0);
    for (size_t p = 0; p < events.size(); p++) {
        if (events[p] < 0) { last[constraints[~events[p]]] = p; continue; }
        const p3gpu_air_node &n = nodes[events[p]];
        if (is_binary(n.op) || n.op == P3GPU_AIR_NEG) last[n.a] = p;
        if (is_binary(n.op)) last[n.b] = p;
    }
    std::vector<u32> slot(n_nodes, 0), free_slots;
    AirProgram prog;
    prog.field = field; prog.width = width; prog.n_public = n_public; prog.n_constraints = (u32)n_constraints;
    prog.pre_width = pre_width; prog.n_periodic = n_periodic;
    prog.insns.reserve(events.size());
    auto release = [&](u32 node, size_t p) { if (last[node] == p) free_slots.push_back(slot[node]); };
    for (size_t p = 0; p < events.size(); p++) {
        if (events[p] < 0) {
            const u32 k = (u32)~events[p], c = constraints[k];
            prog.insns.push_back({AIR_OP_FOLD | (k << 4), slot[c]});
            release(c, p);
            continue;
        }
        const u32 i = (u32)events[p];
        const p3gpu_air_node &n = nodes[i];
        u32 arg = 0, op = n.op;
        switch (n.op) {
            case P3GPU_AIR_CONST: arg = n.imm; break;
            case P3GPU_AIR_MAIN_LOCAL: arg = n.a; break;
            case P3GPU_AIR_MAIN_NEXT: arg = n.a; prog.uses |= AIR_USES_NEXT; break;
            case P3GPU_AIR_PUBLIC: arg = n.a; prog.uses |= AIR_USES_PUBLIC; break;
            case P3GPU_AIR_IS_FIRST_ROW: case P3GPU_AIR_IS_LAST_ROW: case P3GPU_AIR_IS_TRANSITION: prog.uses |= AIR_USES_SELECTORS; break;
            case P3GPU_AIR_PREPROCESSED_LOCAL: arg = n.a; op = AIR_OP_PRE_LOCAL; prog.uses |= AIR_USES_PRE_LOCAL; break;
            case P3GPU_AIR_PREPROCESSED_NEXT: arg = n.a; op = AIR_OP_PRE_NEXT; prog.uses |= AIR_USES_PRE_NEXT; break;
            case P3GPU_AIR_PERIODIC: arg = n.a; op = AIR_OP_PERIODIC; prog.uses |= AIR_USES_PERIODIC; break;
            case P3GPU_AIR_NEG: arg = slot[n.a]; release(n.a, p); break;
            default:
                arg = slot[n.a] | (slot[n.b] << 16);
                release(n.a, p);
                if (n.b != n.a) release(n.b, p);
        }
        if (free_slots.empty()) free_slots.push_back(prog.n_slots++);
        slot[i] = free_slots.back();
        free_slots.pop_back();
        if (prog.n_slots > lim.max_slots)
            return fail(P3GPU_EUNSUPPORTED, "AIR program: more than " + std::to_string(lim.max_slots) + " simultaneously live values (slots)");
        prog.insns.push_back({op | (slot[i] << 4), arg});
    }
    out = std::move(prog);
    return P3GPU_OK;
}

inline int32_t air_compile(int field, const p3gpu_air_node *nodes, size_t n_nodes, const uint32_t *constraints, size_t n_constraints,
                           u32 width, u32 n_public, AirProgram &out, std::string &err) {
    return air_compile(field, nodes, n_nodes, constraints, n_constraints, width, n_public, 0, 0, out, err);
}

// ---- per-instruction semantics and per-row quotient, shared by the kernel and host C++ -------------------------------------
template <int F> __host__ __device__ __forceinline__ void air_qmac(u64 (&acc)[4], u32 c, const uint4 a) {
    // acc += c * a (base x EF4), lazily: invariant acc < p * 2^32 (open.cu lazy_mac)
    const u32 av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
    for (int d = 0; d < 4; d++) {
        acc[d] += (u64)c * av[d];
        u32 hi = (u32)(acc[d] >> 32);
        const u32 hs = hi - Fp<F>::P;
        hi = hi < hs ? hi : hs;
        acc[d] = ((u64)hi << 32) | (u32)acc[d];
    }
}

__host__ __device__ __forceinline__ u32 air_bitrev(u32 i, unsigned bits) {
    if (bits == 0) return 0;
#ifdef __CUDA_ARCH__
    return __brev(i) >> (32 - bits);
#else
    u32 r = 0;
    for (unsigned b = 0; b < bits; b++) r |= ((i >> b) & 1u) << (bits - 1 - b);
    return r;
#endif
}

// Per-launch constants of the quotient evaluation over the quotient domain g * K, |K| = 2^log_q = 2^(log_n + q).
struct AirDomain {
    unsigned log_q, q;          // q = log_q - log_n
    u32 shift;                  // g = GENERATOR (Montgomery)
    u32 w_q;                    // generator of K
    u32 w_n_inv;                // omega_N^-1
    u32 uses;
    u32 periodic_mask;          // rows of the periodic table - 1 (natural index i reads row i & periodic_mask)
};

// Arguments of a hand-written AIR quotient kernel (keccak_air.cu, blake3_air.cu, poseidon1_air.cu), launched by air_hand_quotient
// (air_program.cu): 2N points of GENERATOR * K, |K| = 2N, read from the first 2N rows of the committed bit-reversed LDE.
// A SHARDED instance (blake3_air.cu, sha256_air.cu, poseidon1_air.cu) evaluates one rank's row block of the row-sharded commit
// instead: block row m is memory row row0 + m of the bit-reversed LDE (natural index bitrev(row0 + m)), read in place through the
// unit table (AirShardRow), and its quotient goes to q[m].
struct AirHandQArgs {
    const u32 *lde;            // bit-reversed LDE prefix, >= 2^d.log_q rows x the AIR's width (SHARDED: the rank's row block)
    const uint4 *apow;         // alpha^(K - 1 - k), k < K
    u32 *q;                    // 2^d.log_q x 4, natural order (SHARDED: rows x 4, the block's bit-reversed slice)
    AirDomain d;
    u32 zh[2], izh[2];         // Z_H and 1 / Z_H by i mod 2
    const u32 *consts;         // the AIR's constants on the device, owned by the context (null for AIRs without any)
    u32 lanes;                 // lanes per point: 32 (one warp per point) or the AIR's vector length
    // SHARDED only
    const u64 *units;          // n_units entries of the unit table, one per 8 columns
    u32 n_units, row0, rows;   // the block is memory rows [row0, row0 + rows)
};

// ---- address translation of a row block left chunk-major by p3gpu_commit_sharded_dev ------------------------------------
// The block is a list of column segments, each a (rows x width) row-major matrix (shard_col_segments).  Every segment bound is a
// multiple of AIR_UNIT columns or the trace's end, so each unit of AIR_UNIT columns [8u, 8u + 8) lies in one segment, and the unit
// table holds, per unit, where that segment puts column c of block row m:  base + m * stride + c, with base = offset - first
// column (>= 0: offset = rows * first column) in the low 48 bits and the segment's width (stride) in the high 16.  A load of 2 or 4
// words at an even / 4-aligned column stays inside one unit, so vector loads need no splitting; they are as aligned as in the dense
// matrix, because base and stride are multiples of 8 except in the single segment of a one-rank block (base 0, stride the width).
// A column window of a generated trace (the trace generators' WINDOW instances): only columns [col0, col1) of the rows of vec_len
// permutations (or of one hash per row, vec_len 1) are stored, as a dense rows x (col1 - col0) matrix.
struct GenWindow { size_t col0, col1; unsigned vec_len; };

constexpr u32 AIR_UNIT = 8;
constexpr u64 AIR_UNIT_BASE_MASK = (1ull << 48) - 1;
inline u64 air_unit_entry(u64 base, u64 stride) { return base | (stride << 48); }

#ifdef __CUDACC__
// the unit table into shared memory (before the block's __syncthreads)
__device__ __forceinline__ void air_shard_table_load(const AirHandQArgs &a, u64 *tab) {
    for (u32 t = threadIdx.x; t < a.n_units; t += blockDim.x) tab[t] = __ldg(a.units + t);
}
#endif
// block row m of a row block, read through the unit table (shared memory on the device; host C++ runs the same arithmetic)
struct AirShardRow {
    const u32 *blk;
    const u64 *tab;
    u32 m;
    __host__ __device__ __forceinline__ const u32 *at(u32 c) const {
        const u64 e = tab[c / AIR_UNIT];
        return blk + (e & AIR_UNIT_BASE_MASK) + (size_t)m * (u32)(e >> 48) + c;
    }
    __host__ __device__ __forceinline__ u32 ld(u32 c) const {
#ifdef __CUDA_ARCH__
        return __ldg(at(c));
#else
        return *at(c);
#endif
    }
};

// ---- where a point's rows live in the row-sharded commit ------------------------------------------------------------------
// Rank g holds memory rows [g R, (g + 1) R) of the bit-reversed LDE, R = 2^log_rows: memory row M is local row M mod R of rank
// M / R.  Point i = bitrev(M) reads its next row at natural index i + 2^q, memory row bitrev(i + 2^q).  The owner of a memory row
// is its top log2(G) bits, i.e. the low log2(G) bits of the natural index; those are bitrev(g) for every point of rank g, and adding
// 2^q changes them the same way for all of them (a carry only leaves upwards).  So every next row of rank g lies on ONE rank,
// bitrev((bitrev(g) + 2^q) mod G), which is g itself when G <= 2^q.
struct AirShardLoc { u32 rank, row; };
__host__ __device__ __forceinline__ AirShardLoc air_shard_locate(u32 mem_row, unsigned log_rows) {
    return AirShardLoc{mem_row >> log_rows, mem_row & ((1u << log_rows) - 1u)};
}
__host__ __device__ __forceinline__ u32 air_shard_next_rank(u32 rank, unsigned log_world, unsigned q) {
    if (q >= log_world) return rank;
    const u32 mask = (1u << log_world) - 1u;
    return air_bitrev((air_bitrev(rank, log_world) + (1u << q)) & mask, log_world);
}

// selectors_on_coset (commit/src/domain.rs:321-361) at x_i = g * w_q^i, unnormalised: Z_H / (x - 1), Z_H / (x - w^-1), x - w^-1.
// zh = Z_H(x_i).  Shared by the constraint-program kernel and the hand-written Keccak AIR kernel (keccak_air.cu).
template <int F> __host__ __device__ __forceinline__ void air_selectors(const AirDomain &d, u32 i, u32 zh, u32 &first, u32 &last, u32 &trans) {
    const u32 x = mont_mul<F>(d.shift, fp_pow<F>(d.w_q, i));
    const u32 a = fp_sub<F>(x, Fp<F>::ONE), b = fp_sub<F>(x, d.w_n_inv);
    const u32 inv_ab = fp_inv<F>(mont_mul<F>(a, b));          // one inversion for both denominators
    first = mont_mul<F>(zh, mont_mul<F>(b, inv_ab));
    last = mont_mul<F>(zh, mont_mul<F>(a, inv_ab));
    trans = b;
}

#ifdef __CUDACC__
// ---- device helpers of the hand-written quotient kernels ------------------------------------------------------------------
template <int F> __device__ __forceinline__ u32 air_bxor(u32 x, u32 y) { return fp_sub<F>(fp_add<F>(x, y), fp_double<F>(mont_mul<F>(x, y))); }   // x + y - 2xy
template <int F> __device__ __forceinline__ u32 air_bool(u32 x) { return mont_mul<F>(x, fp_sub<F>(x, Fp<F>::ONE)); }                         // x (x - 1)

// The end of a warp's point: reduce every lane's lazy accumulators, add them over the 32 lanes, multiply by 1 / Z_H(x_nat) and let
// lanes 0..3 store the four coefficients of q[i].  1 / Z_H depends on the natural index nat's parity only: `odd` = nat & 1.
template <int F> __device__ __forceinline__ void air_warp_store(const AirHandQArgs &a, const u64 (&acc)[4], u32 i, unsigned lane, u32 odd) {
    u32 r[4];
#pragma unroll
    for (int d = 0; d < 4; d++) r[d] = mont_redc<F>(acc[d]);
#pragma unroll
    for (int o = 16; o; o >>= 1)
#pragma unroll
        for (int d = 0; d < 4; d++) r[d] = fp_add<F>(r[d], __shfl_xor_sync(0xffffffffu, r[d], o));
    const u32 mine = lane == 0 ? r[0] : lane == 1 ? r[1] : lane == 2 ? r[2] : r[3];
    if (lane < 4) a.q[4 * (size_t)i + lane] = mont_mul<F>(mine, odd ? a.izh[1] : a.izh[0]);
}
template <int F> __device__ __forceinline__ void air_warp_store(const AirHandQArgs &a, const u64 (&acc)[4], u32 i, unsigned lane) {
    air_warp_store<F>(a, acc, i, lane, i & 1u);
}

// The natural index of SHARDED block row m: bitrev(row0 + m) over the 2^log_q-point domain; its parity is the top bit of row0 + m.
__device__ __forceinline__ u32 air_shard_odd(const AirHandQArgs &a, u32 m) { return ((a.row0 + m) >> (a.d.log_q - 1)) & 1u; }
#endif

// Decodes one instruction: every opcode but FOLD computes its value into v and returns false, for the caller to store in slot dst;
// a FOLD returns true and is the caller's (the quotient accumulates it against an alpha power, the check tests it for zero).  The
// one copy of each opcode's semantics.  Env supplies slot(s), local(c), next(c), pub(k) and, with EXT (opcodes 12-14), pre_local(c), pre_next(c) and
// periodic(k); first / last / trans are the selectors' values at the row.
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <int F, bool EXT, class Env>
__host__ __device__ __forceinline__ bool air_decode(Env &env, const AirInsn in, u32 first, u32 last, u32 trans, u32 &v) {
    const u32 op = in.op_dst & 15u;
    switch (op) {
        case P3GPU_AIR_CONST: v = in.arg; break;
        case P3GPU_AIR_MAIN_LOCAL: v = env.local(in.arg); break;
        case P3GPU_AIR_MAIN_NEXT: v = env.next(in.arg); break;
        case P3GPU_AIR_PUBLIC: v = env.pub(in.arg); break;
        case P3GPU_AIR_IS_FIRST_ROW: v = first; break;
        case P3GPU_AIR_IS_LAST_ROW: v = last; break;
        case P3GPU_AIR_IS_TRANSITION: v = trans; break;
        case P3GPU_AIR_ADD: v = fp_add<F>(env.slot(in.arg & 0xffffu), env.slot(in.arg >> 16)); break;
        case P3GPU_AIR_SUB: v = fp_sub<F>(env.slot(in.arg & 0xffffu), env.slot(in.arg >> 16)); break;
        case P3GPU_AIR_NEG: v = fp_neg<F>(env.slot(in.arg)); break;
        case P3GPU_AIR_MUL: v = mont_mul<F>(env.slot(in.arg & 0xffffu), env.slot(in.arg >> 16)); break;
        default:                                                    // AIR_OP_FOLD (and, with EXT, opcodes 12-14)
            if constexpr (EXT) {
                if (op != AIR_OP_FOLD) {
                    v = op == AIR_OP_PRE_LOCAL ? env.pre_local(in.arg) : op == AIR_OP_PRE_NEXT ? env.pre_next(in.arg) : env.periodic(in.arg);
                    break;
                }
            }
            return true;
    }
    return false;
}

// Evaluates the program at natural index i.  Env supplies insn(pc), slot(s), local(c), next(c), pub(k), apow(k) (alpha^(K-1-k)),
// the row loads for memory rows bitrev(i) / bitrev(i + 2^q), zh(i) = Z_H(x_i) and inv_zh(i).  EXT (a program that reads
// preprocessed or periodic columns) compiles in opcodes 12-14: Env then also supplies set_ext_rows(m, m_next, periodic_row),
// pre_local(c), pre_next(c) and periodic(k).  Without EXT those opcodes and row pointers do not exist in the instance.
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <int F, bool EXT = false, class Env>
__host__ __device__ __forceinline__ uint4 air_row_quotient(Env &env, const AirDomain &d, u32 n_insns, u32 i) {
    const u32 mask = d.log_q == 32 ? 0xffffffffu : ((1u << d.log_q) - 1u);
    const u32 next_uses = EXT ? (AIR_USES_NEXT | AIR_USES_PRE_NEXT) : AIR_USES_NEXT;
    const u32 m = air_bitrev(i, d.log_q), mn = (d.uses & next_uses) ? air_bitrev((i + (1u << d.q)) & mask, d.log_q) : 0u;
    env.set_rows(m, mn);
    if constexpr (EXT) env.set_ext_rows(m, mn, i & d.periodic_mask);
    u32 first = 0, last = 0, trans = 0;
    if (d.uses & AIR_USES_SELECTORS) air_selectors<F>(d, i, env.zh(i), first, last, trans);
    u64 acc[4] = {0, 0, 0, 0};
    for (u32 pc = 0; pc < n_insns; pc++) {
        const AirInsn in = env.insn(pc);
        const u32 dst = in.op_dst >> 4;
        u32 v;
        if (air_decode<F, EXT>(env, in, first, last, trans, v)) {
            air_qmac<F>(acc, env.slot(in.arg), env.apow(dst));
            continue;
        }
        env.slot(dst) = v;
    }
    const u32 z = env.inv_zh(i);
    return make_uint4(mont_mul<F>(mont_redc<F>(acc[0]), z), mont_mul<F>(mont_redc<F>(acc[1]), z), mont_mul<F>(mont_redc<F>(acc[2]), z),
                      mont_mul<F>(mont_redc<F>(acc[3]), z));
}

// Checks row i of a trace of `height` rows (any height >= 1) with the reference's debug semantics (air/src/check_constraints.rs):
// the trace in natural row order, next row (i + 1) mod height for the main and the preprocessed trace, selectors [i = 0],
// [i = height - 1] and [i != height - 1] as Montgomery 0 / 1, periodic row i mod periodic_rows.  Calls on_fail(k) for every
// constraint k whose value is non-zero, in ascending k (the compiler emits the folds in assertion order).  Env supplies what
// air_decode reads for the EXT instance, insn(pc), set_rows(i, i_next) and set_ext_rows(i, i_next, periodic_row).
#ifdef __CUDACC__
#pragma nv_exec_check_disable
#endif
template <int F, class Env, class OnFail>
__host__ __device__ __forceinline__ void air_row_check(Env &env, u32 n_insns, u32 i, u32 height, u32 periodic_rows, OnFail &on_fail) {
    const bool is_last = i + 1 == height;
    const u32 nxt = is_last ? 0u : i + 1;
    env.set_rows(i, nxt);
    env.set_ext_rows(i, nxt, periodic_rows > 1 ? i % periodic_rows : 0u);
    const u32 first = i == 0 ? Fp<F>::ONE : 0u, last = is_last ? Fp<F>::ONE : 0u, trans = is_last ? 0u : Fp<F>::ONE;
    for (u32 pc = 0; pc < n_insns; pc++) {
        const AirInsn in = env.insn(pc);
        const u32 dst = in.op_dst >> 4;
        u32 v;
        if (air_decode<F, true>(env, in, first, last, trans, v)) {
            if (env.slot(in.arg) != 0u) on_fail(dst);
            continue;
        }
        env.slot(dst) = v;
    }
}

// Host-side launch constants + tables: Z_H(x_i) and 1/Z_H(x_i) depend on i mod 2^q only (x^N = g^N w_q^(iN), w_q^N of order 2^q).
template <int F> inline AirDomain air_domain(unsigned log_q, unsigned log_n, u32 uses, std::vector<u32> &zh, std::vector<u32> &inv_zh) {
    AirDomain d;
    d.log_q = log_q; d.q = log_q - log_n; d.uses = uses; d.periodic_mask = 0;
    d.shift = to_monty<F>(Fp<F>::GEN);
    d.w_q = two_adic_generator<F>(log_q);
    d.w_n_inv = fp_inv<F>(two_adic_generator<F>(log_n));
    const size_t nz = (size_t)1 << d.q;
    zh.resize(nz); inv_zh.resize(nz);
    const u32 s_pow_n = fp_pow<F>(d.shift, (u64)1 << log_n), wr = two_adic_generator<F>(d.q);
    u32 wp = Fp<F>::ONE;
    for (size_t j = 0; j < nz; j++) {
        zh[j] = fp_sub<F>(mont_mul<F>(s_pow_n, wp), Fp<F>::ONE);
        inv_zh[j] = fp_inv<F>(zh[j]);
        wp = mont_mul<F>(wp, wr);
    }
    return d;
}

// alpha^(K - 1 - k) for k < K, as the kernel's shared table holds it
template <int F> inline std::vector<uint4> air_alpha_table(const u32 alpha[4], u32 K) {
    std::vector<uint4> t(K);
    Ef4<F> cur, al;
    cur.c[0] = Fp<F>::ONE; cur.c[1] = cur.c[2] = cur.c[3] = 0;
    for (int j = 0; j < 4; j++) al.c[j] = alpha[j];
    for (u32 j = 0; j < K; j++) {
        t[K - 1 - j] = make_uint4(cur.c[0], cur.c[1], cur.c[2], cur.c[3]);
        cur = ef_mul<F>(cur, al);
    }
    return t;
}

}  // namespace p3
