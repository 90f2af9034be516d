// Internal declarations shared by the translation units of libp3gpu.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/p3gpu.h"
#include "field.cuh"
#include "poseidon2_consts.h"

namespace p3 {

void set_error(const char *fmt, ...);

#define P3_CUDA(call)                                                                           \
    do {                                                                                        \
        cudaError_t e__ = (call);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            p3::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return P3GPU_ECUDA;                                                                 \
        }                                                                                       \
    } while (0)

#define P3_CHECK(cond, code, ...)                 \
    do {                                          \
        if (!(cond)) {                            \
            p3::set_error(__VA_ARGS__);           \
            return (code);                        \
        }                                         \
    } while (0)

// first statement of every extern "C" entry point that takes a context: serialise callers, select the device (CUDA's current
// device is per host thread: callers may come from any thread)
#define P3_ENTER(ctx)                                                        \
    P3_CHECK((ctx) != nullptr, P3GPU_EINVAL, "null context");                \
    std::lock_guard<std::recursive_mutex> p3_lock__((ctx)->call_mu);         \
    P3_CUDA(cudaSetDevice((ctx)->device));                                   \
    (ctx)->tick++

#define P3_TRY(expr)                      \
    do {                                  \
        int32_t rc__ = (expr);            \
        if (rc__ != P3GPU_OK) return rc__; \
    } while (0)


struct TwiddleKey {
    int field, log_n; u32 shift; int inverse;
    bool operator<(const TwiddleKey &o) const {
        return std::tie(field, log_n, shift, inverse) < std::tie(o.field, o.log_n, o.shift, o.inverse);
    }
};

}  // namespace p3

namespace p3 { struct TwiddleEntry { uint2 *ptr; size_t bytes; uint64_t last_use; }; }

struct p3gpu_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t switch_event = nullptr;   // orders work across p3gpu_ctx_set_stream changes (shared scratch / caches)
    int sm_count = 132;                   // H100 SXM; replaced by the device's count in p3gpu_ctx_create
    uint64_t launches = 0;
    // Every extern "C" entry point holds call_mu for its whole duration: the reference's objects are Clone + Sync and may be
    // called through &self from several threads (SURVEY 8b "Threading"); a context serialises such callers (scratch buffers,
    // caches and the stream are per context).  Clones that want concurrency create their own context.
    std::recursive_mutex call_mu;
    uint64_t tick = 0;                    // entry-point counter: LRU clock of the twiddle cache
    // twiddle heaps keyed like the reference's coset_twiddles cache (radix_2_dit_parallel.rs:32-40), bounded by bytes (LRU)
    std::map<p3::TwiddleKey, p3::TwiddleEntry> twiddles;
    size_t twiddle_bytes = 0;
    size_t twiddle_cap_bytes = (size_t)2 << 30;   // P3GPU_TWIDDLE_CACHE_MB
    void *leaf_table = nullptr; size_t leaf_table_bytes = 0;
    // host-pointer entry points: copy streams + events of the chunked H2D || compute || D2H pipeline, double-buffered chunk buffers
    cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;
    cudaEvent_t ev_h2d[2] = {nullptr, nullptr}, ev_comp[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr}, ev_start = nullptr;
    void *chunk_in[2] = {nullptr, nullptr}; size_t chunk_in_bytes[2] = {0, 0};
    void *chunk_out[2] = {nullptr, nullptr}; size_t chunk_out_bytes[2] = {0, 0};
    // staged multi-GPU exchange: staging buffers (one LDE'd column chunk each), exchange stream and events
    cudaStream_t xchg_stream = nullptr;
    cudaStream_t dma_stream[16] = {nullptr}; cudaEvent_t dma_done[16] = {nullptr};   // dma exchange: one copy stream per destination rank
    cudaEvent_t ev_stage_full[2] = {nullptr, nullptr}, ev_stage_free[2] = {nullptr, nullptr};
    void *stage_buf[2] = {nullptr, nullptr}; size_t stage_bytes[2] = {0, 0};   // device copy of the per-height matrix table (> 8 matrices)
    // FRI half-inverse-power tables (bit-reversed), one per field, grown on demand
    uint32_t *fold_table[2] = {nullptr, nullptr};
    size_t fold_table_len[2] = {0, 0};
    // grow-only scratch
    void *scratch = nullptr; size_t scratch_bytes = 0;
    void *scratch2 = nullptr; size_t scratch2_bytes = 0;
    void *lde_tiles = nullptr; size_t lde_tiles_bytes = 0;   // coset LDE: the fused pass's tile-major output (ntt.cu), used by nothing else
    void *pool[4] = {nullptr, nullptr, nullptr, nullptr}; size_t pool_bytes[4] = {0, 0, 0, 0};  // host-pointer wrappers / commit phase
    // Poseidon2 constants: [field][0: width 16, 1: width 24], host copy + device copy
    p3::Poseidon2Consts p2_host[2][2];
    p3::Poseidon2Consts *p2_dev = nullptr;  // 4 entries
    alignas(8) unsigned char air_consts[1024];   // Poseidon2 AIR round constants (air.cu: AirConsts)
    int air_field = -1;                          // the field they were set for (-1: not set)
    // Poseidon1 AIR constants (poseidon1_air.cu): a device buffer of this context, written by p3gpu_p1air_set_constants on the
    // context's stream, freed at destroy; p1_field is the field they were set for (-1: not set)
    uint32_t *p1_consts = nullptr;
    int p1_field = -1, p1_rounds_p = 0;
};

namespace p3 {

int32_t ctx_scratch(p3gpu_ctx *ctx, size_t bytes, void **out);
int32_t ctx_scratch2(p3gpu_ctx *ctx, size_t bytes, void **out);
int32_t ctx_lde_tiles(p3gpu_ctx *ctx, size_t bytes, void **out);
int32_t ctx_pool(p3gpu_ctx *ctx, int slot, size_t bytes, void **out);
int32_t ctx_leaf_table(p3gpu_ctx *ctx, size_t bytes, void **out);  // grow-only cached device buffers (no malloc/free per call)

// ntt.cu
int32_t ntt_dft_batch(p3gpu_ctx *ctx, int field, int kind, const u32 *d_in, u32 *d_out, size_t h, size_t w, u32 shift);
int32_t ntt_coset_lde(p3gpu_ctx *ctx, int field, const u32 *d_in, size_t h, size_t w, unsigned added_bits, u32 shift,
                      u32 *d_out, int bitrev_rows, size_t in_pitch = 0, size_t out_pitch = 0);
int32_t ntt_lde_coefficients(p3gpu_ctx *ctx, int field, u32 *d_trace, size_t h, size_t w);
int32_t ntt_lde_coset_block(p3gpu_ctx *ctx, int field, const u32 *d_coef, size_t h, size_t w, unsigned added_bits, u32 shift, size_t coset,
                            u32 *d_out);
// hash.cu
int32_t hash_poseidon2_permute(p3gpu_ctx *ctx, int field, int width, u32 *d_states, size_t n);
int32_t hash_keccak_f(p3gpu_ctx *ctx, u64 *d_states, size_t n);
int32_t hash_merkle_commit(p3gpu_ctx *ctx, int field, int hash, size_t n_mats, const u32 *const *d_mats,
                           const size_t *heights, const size_t *widths, u32 *d_layers, size_t *layer_lens,
                           size_t *n_layers);
int32_t hash_merkle_from_digests(p3gpu_ctx *ctx, int field, int hash, const u32 *d_digests, size_t n, u32 *d_layers,
                                 size_t *layer_lens, size_t *n_layers);
// fri.cu
int32_t fri_fold(p3gpu_ctx *ctx, int field, const u32 *d_in, size_t rows, unsigned log_arity, const u32 beta[4], u32 *d_out);

int32_t fri_ef_axpy(p3gpu_ctx *ctx, int field, u32 *d_acc, const u32 *d_x, size_t n, const u32 s[4]);

// open.cu
int32_t open_inv_denoms(p3gpu_ctx *ctx, int field, unsigned log_h, const u32 *z, const u32 *zinv, u32 *d_out, u32 *d_adj);
int32_t open_columnwise_dot(p3gpu_ctx *ctx, int field, const u32 *d_mat, size_t h, size_t w, const u32 *d_vec, u32 *d_out, const u32 *scale);
int32_t open_rowwise_dot(p3gpu_ctx *ctx, int field, const u32 *d_mat, size_t h, size_t w, const u32 *alpha, u32 *d_out);
int32_t open_reduce(p3gpu_ctx *ctx, int field, u32 *d_ro, const u32 *d_r, const u32 *d_invd, size_t h, const u32 *coeff, const u32 *yred);

// ntt.cu / peer.cu: multi-GPU
int32_t ntt_coset_lde_sharded(p3gpu_ctx *ctx, int field, const u32 *d_in, size_t h, size_t w_local, unsigned added_bits, u32 shift,
                              unsigned world, u32 *const *rank_out, size_t w_total, size_t col_off, int chunk_major = 0);
std::vector<size_t> shard_chunk_bounds(size_t w_local);
int32_t peer_push_rows(p3gpu_ctx *ctx, cudaStream_t stream, unsigned world, u32 *const *rows, const u32 *d_src, size_t H, size_t wc, size_t w_total,
                       size_t dst_col, unsigned log_rows);
int32_t peer_barrier(p3gpu_ctx *ctx, unsigned world, unsigned rank, void *const *ctrl, u32 epoch, double timeout_s);
int32_t peer_allgather(p3gpu_ctx *ctx, unsigned world, unsigned rank, void *const *tables, const u32 *d_src, size_t words);

// air.cu: Poseidon2 AIR trace generation / quotient (SURVEY 8f ranks 2-3)
size_t air_columns(int field, int rounds_p);            // 0 for an unknown field
int32_t air_set_constants(p3gpu_ctx *ctx, int field, const u32 *beg, const u32 *part, int rounds_p, const u32 *end);
int32_t air_generate_trace(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_perms, u32 *d_trace);
int32_t air_quotient(p3gpu_ctx *ctx, int field, int vec_len, const u32 *d_lde, unsigned log_h, unsigned log_n, const u32 *alpha, u32 *d_q);
int32_t air_sharded_field(int field);                   // P3GPU_EUNSUPPORTED for BabyBear: the sharded entry points are KoalaBear-only
int32_t air_generate_trace_cols(p3gpu_ctx *ctx, int field, int vec_len, const u32 *d_inputs, size_t n_perms, size_t col0, size_t col1, u32 *d_out);
int32_t shard_col_segments(unsigned world, const size_t *col_starts, size_t rows, std::vector<size_t> &segs);   // (c0, c1, offset) triples
int32_t air_quotient_sharded(p3gpu_ctx *ctx, int field, int vec_len, unsigned world, unsigned rank, const u32 *d_block, const size_t *col_starts,
                             unsigned log_h, unsigned log_n, const u32 *alpha, u32 *d_q);

// air_program.cu: any AIR as a constraint program (air_program.cuh)
// check: a check program (air_check.cu), compiled under the check limits (air_program.cuh AIR_CHECK_LIMITS)
int32_t air_program_create(p3gpu_ctx *ctx, int field, const p3gpu_air_node *nodes, size_t n_nodes, const u32 *constraints, size_t n_constraints,
                           const p3gpu_air_layout &layout, p3gpu_air_program **out, bool check = false);
void air_program_destroy(p3gpu_air_program *prog);
int32_t air_program_info(const p3gpu_air_program *prog, size_t *n_insns, size_t *n_slots, size_t *n_cons);
// layout_entry: called through p3gpu_air_quotient_layout_dev (d_pre / d_periodic as the program's layout declares them); otherwise
// through p3gpu_air_quotient_dev, which refuses a program with preprocessed or periodic columns
int32_t air_program_quotient(p3gpu_ctx *ctx, const p3gpu_air_program *prog, const u32 *d_lde, unsigned log_lde, const u32 *d_pre,
                             unsigned log_pre, const u32 *d_periodic, unsigned log_periodic_rows, unsigned log_q, unsigned log_n,
                             const u32 *pubs, const u32 *alpha, u32 *d_q, bool layout_entry);
// rank `rank`'s row block rows[rank] of the row-sharded commit with column blocks col_starts (p3gpu_air_quotient_sharded_dev);
// rows: every rank's row block (the peer blocks are read for next-row columns)
int32_t air_program_quotient_sharded(p3gpu_ctx *ctx, const p3gpu_air_program *prog, unsigned world, unsigned rank, u32 *const *rows,
                                     const size_t *col_starts, const u32 *d_periodic, unsigned log_periodic_rows, unsigned log_lde, unsigned log_n,
                                     const u32 *pubs, const u32 *alpha, u32 *d_q);
// air_check.cu: the debug constraint check of a check program over the trace domain; pass 1 writes d_counts (height words), pass 2
// (d_counts null) the failing constraints of the n_rows listed rows at their offsets
int32_t air_check(p3gpu_ctx *ctx, const p3gpu_air_program *pg, const u32 *d_trace, size_t height, const u32 *d_pre, const u32 *d_periodic,
                  size_t periodic_rows, const u32 *pubs, u32 *d_counts, const u32 *d_rows, size_t n_rows, const u64 *d_offsets, u32 *d_failed);
// A hand-written AIR quotient kernel (AirHandQArgs, air_program.cuh) over the 2N points of GENERATOR * K from the first 2N rows of
// the committed bit-reversed LDE: checks the field, the domain, the alignment and alpha (messages name the AIR), builds the domain
// and the alpha^(K - 1 - k) table (scratch2), then launches `kern_<field>` on min(SMs, 2N lanes / (32 warps)) blocks of `warps`
// warps.  `lanes`: lanes per point (32: one warp per point); `consts`: the AIR's device constants, handed to the kernel.
// `shard` (sharded mode, the kernels' SHARDED instances): d_lde is rank `rank`'s row block of the row-sharded commit of a `width`-column
// trace over `world` ranks with column blocks `col_starts` (log_lde = log_n + 1, R = 2N / world rows), d_q its R x 4 bit-reversed
// quotient slice; the unit table (air_program.cuh AirShardRow) goes behind the alpha table, `smem` grows by its size.
struct AirHandShard { unsigned world, rank; const size_t *col_starts; size_t width; };
int32_t air_hand_quotient(p3gpu_ctx *ctx, int field, const char *name, const void *kern_babybear, const void *kern_koalabear, u32 n_constraints,
                          unsigned warps, size_t smem, u32 uses, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q,
                          const u32 *consts = nullptr, unsigned lanes = 32, const AirHandShard *shard = nullptr);
// The unit table of a row block (air_program.cuh AirShardRow): one entry per 8 columns of the `width`-column trace, from
// shard_col_segments; EINVAL when a segment bound is neither a multiple of 8 columns nor the trace's end.
int32_t air_shard_units(unsigned world, const size_t *col_starts, size_t rows, size_t width, std::vector<u64> &units);
// A trace generator's column window [col0, col1) of a `width`-column trace: EINVAL unless col0 <= col1 <= width
int32_t air_check_window(const char *name, size_t col0, size_t col1, size_t width);

// keccak_air.cu: Keccak-f AIR trace generation / quotient
size_t keccak_air_height(size_t n_hashes);
int32_t keccak_air_generate(p3gpu_ctx *ctx, int field, const u64 *d_inputs, size_t n_hashes, u32 *d_trace);
int32_t keccak_air_quotient(p3gpu_ctx *ctx, int field, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q);

// blake3_air.cu: Blake3 AIR trace generation / quotient
int32_t blake3_air_generate(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, u32 *d_trace);
int32_t blake3_air_quotient(p3gpu_ctx *ctx, int field, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q);
int32_t blake3_air_generate_cols(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, size_t col0, size_t col1, u32 *d_out);
int32_t blake3_air_quotient_sharded(p3gpu_ctx *ctx, int field, const AirHandShard &shard, const u32 *d_block, unsigned log_lde, unsigned log_n,
                                    const u32 *alpha, u32 *d_q);

// sha256_air.cu: SHA-256 AIR trace generation / quotient
int32_t sha256_air_generate(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, u32 *d_trace);
int32_t sha256_air_quotient(p3gpu_ctx *ctx, int field, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q);
int32_t sha256_air_generate_cols(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_hashes, size_t col0, size_t col1, u32 *d_out);
int32_t sha256_air_quotient_sharded(p3gpu_ctx *ctx, int field, const AirHandShard &shard, const u32 *d_block, unsigned log_lde, unsigned log_n,
                                    const u32 *alpha, u32 *d_q);

// poseidon1_air.cu: Poseidon1 AIR constants (per context), trace generation / quotient
size_t p1air_columns(int field, int rounds_p);          // 0 for an unknown field
int32_t p1air_set_constants(p3gpu_ctx *ctx, int field, const u32 *initial_full, const u32 *terminal_full, const u32 *mds_circ_col,
                            const u32 *first_round_constants, const u32 *m_i, const u32 *partial_rc, const u32 *sparse_first_row, const u32 *v,
                            int rounds_p);
int32_t p1air_generate(p3gpu_ctx *ctx, int field, const u32 *d_inputs, size_t n_perms, u32 *d_trace);
int32_t p1air_quotient(p3gpu_ctx *ctx, int field, int vector_len, const u32 *d_lde, unsigned log_lde, unsigned log_n, const u32 *alpha, u32 *d_q);
int32_t p1air_generate_cols(p3gpu_ctx *ctx, int field, int vector_len, const u32 *d_inputs, size_t n_perms, size_t col0, size_t col1, u32 *d_out);
int32_t p1air_quotient_sharded(p3gpu_ctx *ctx, int field, int vector_len, const AirHandShard &shard, const u32 *d_block, unsigned log_lde,
                               unsigned log_n, const u32 *alpha, u32 *d_q);

// challenger.cu / query.cu: transcript + query-phase gathers of the prove driver (SURVEY 8f rank 4, N1)
int32_t challenger_new(p3gpu_ctx *ctx, int field, int width, int rate, p3gpu_challenger **out);
void challenger_free(p3gpu_ctx *ctx, p3gpu_challenger *ch);
int32_t challenger_clone(p3gpu_ctx *ctx, const p3gpu_challenger *src, p3gpu_challenger **out);
int32_t challenger_observe_dev(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *d_vals, size_t n);
int32_t challenger_observe_host(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *h_vals, size_t n);
int32_t challenger_sample(p3gpu_ctx *ctx, p3gpu_challenger *ch, u32 *h_out, size_t n);
int32_t challenger_grind(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, u32 *witness_monty);
int32_t challenger_new_keccak256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out);
int32_t challenger_new_sha256(p3gpu_ctx *ctx, int field, p3gpu_challenger **out);
int32_t challenger_observe_digest(p3gpu_ctx *ctx, p3gpu_challenger *ch, const u32 *h_words, size_t n);
int32_t challenger_sample_bits(p3gpu_ctx *ctx, p3gpu_challenger *ch, unsigned bits, size_t n, u32 *h_out);
int32_t query_gather_rows(p3gpu_ctx *ctx, const u32 *d_mat, size_t h, size_t w, const u32 *h_idx, size_t n, unsigned shift, u32 *d_out);
int32_t query_merkle_paths(p3gpu_ctx *ctx, const u32 *d_layers, const size_t *layer_lens, size_t n_layers, size_t path_len, const u32 *h_idx,
                           size_t n, unsigned shift, u32 *d_out);

static inline unsigned log2_floor(size_t x) { unsigned l = 0; while ((x >> l) > 1) l++; return l; }
static inline bool is_pow2(size_t x) { return x && !(x & (x - 1)); }

}  // namespace p3
