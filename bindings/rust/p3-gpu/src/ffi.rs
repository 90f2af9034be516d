//! `extern "C"` declarations of `include/p3gpu.h`.
use core::ffi::{c_char, c_int, c_uint, c_void};

#[repr(C)]
pub struct P3GpuCtx {
    _private: [u8; 0],
}

#[repr(C)]
pub struct P3GpuChallenger {
    _private: [u8; 0],
}

#[repr(C)]
pub struct P3GpuAirProgram {
    _private: [u8; 0],
}

/// `p3gpu_air_node`: op is one of the `P3GPU_AIR_*` codes below; operands refer only to earlier nodes.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct P3GpuAirNode {
    pub op: u32,
    pub a: u32,
    pub b: u32,
    pub imm: u32,
}

pub const P3GPU_AIR_CONST: u32 = 0;
pub const P3GPU_AIR_MAIN_LOCAL: u32 = 1;
pub const P3GPU_AIR_MAIN_NEXT: u32 = 2;
pub const P3GPU_AIR_PUBLIC: u32 = 3;
pub const P3GPU_AIR_IS_FIRST_ROW: u32 = 4;
pub const P3GPU_AIR_IS_LAST_ROW: u32 = 5;
pub const P3GPU_AIR_IS_TRANSITION: u32 = 6;
pub const P3GPU_AIR_ADD: u32 = 7;
pub const P3GPU_AIR_SUB: u32 = 8;
pub const P3GPU_AIR_NEG: u32 = 9;
pub const P3GPU_AIR_MUL: u32 = 10;
pub const P3GPU_AIR_PREPROCESSED_LOCAL: u32 = 16;
pub const P3GPU_AIR_PREPROCESSED_NEXT: u32 = 17;
pub const P3GPU_AIR_PERIODIC: u32 = 18;
pub const P3GPU_KECCAK_AIR_COLS: usize = 2633;
pub const P3GPU_BLAKE3_AIR_COLS: usize = 9168;
pub const P3GPU_SHA256_AIR_COLS: usize = 7728;

/// `p3gpu_air_layout`: what a constraint program's leaves may read.
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct P3GpuAirLayout {
    pub width: u32,
    pub n_public: u32,
    pub preprocessed_width: u32,
    pub n_periodic: u32,
}

pub const P3GPU_BABY_BEAR: i32 = 0;
pub const P3GPU_KOALA_BEAR: i32 = 1;
pub const P3GPU_DFT: i32 = 0;
pub const P3GPU_IDFT: i32 = 1;
pub const P3GPU_COSET_DFT: i32 = 2;
pub const P3GPU_COSET_IDFT: i32 = 3;
pub const P3GPU_HASH_POSEIDON2_W16: i32 = 0;
pub const P3GPU_HASH_POSEIDON2_W24: i32 = 1;
pub const P3GPU_HASH_KECCAK: i32 = 2;
pub const P3GPU_HASH_SHA256: i32 = 3;
pub const P3GPU_HASH_SHA256_COMPRESS: i32 = 4;

#[repr(C)]
pub struct P3GpuPeerGroup {
    pub world: u32,
    pub rank: u32,
    pub ctrl: [*mut c_void; 16],
    pub rows: [*mut u32; 16],
    pub timeout_s: f64,
}

unsafe extern "C" {
    pub fn p3gpu_ctx_create(device: c_int, out: *mut *mut P3GpuCtx) -> i32;
    pub fn p3gpu_ctx_destroy(ctx: *mut P3GpuCtx);
    pub fn p3gpu_ctx_sync(ctx: *mut P3GpuCtx) -> i32;
    pub fn p3gpu_last_error() -> *const c_char;
    pub fn p3gpu_malloc(ctx: *mut P3GpuCtx, bytes: usize, dptr: *mut *mut c_void) -> i32;
    pub fn p3gpu_free(ctx: *mut P3GpuCtx, dptr: *mut c_void) -> i32;
    pub fn p3gpu_memcpy_h2d(ctx: *mut P3GpuCtx, dst: *mut c_void, src: *const c_void, bytes: usize) -> i32;
    pub fn p3gpu_memcpy_d2h(ctx: *mut P3GpuCtx, dst: *mut c_void, src: *const c_void, bytes: usize) -> i32;
    pub fn p3gpu_host_register(ptr: *mut c_void, bytes: usize) -> i32;
    pub fn p3gpu_host_unregister(ptr: *mut c_void) -> i32;

    // TwoAdicSubgroupDft
    pub fn p3gpu_dft_batch(ctx: *mut P3GpuCtx, field: c_int, kind: c_int, inout: *mut u32, h: usize, w: usize, shift: u32) -> i32;
    pub fn p3gpu_dft_batch_dev(ctx: *mut P3GpuCtx, field: c_int, kind: c_int, d_in: *const u32, d_out: *mut u32, h: usize, w: usize, shift: u32) -> i32;
    pub fn p3gpu_coset_lde_batch(ctx: *mut P3GpuCtx, field: c_int, input: *const u32, h: usize, w: usize, added_bits: c_uint, shift: u32,
                                 out: *mut u32, bitrev_rows: c_int) -> i32;
    pub fn p3gpu_coset_lde_batch_dev(ctx: *mut P3GpuCtx, field: c_int, d_in: *const u32, h: usize, w: usize, added_bits: c_uint, shift: u32,
                                     d_out: *mut u32, bitrev_rows: c_int) -> i32;
    pub fn p3gpu_lde_coefficients_dev(ctx: *mut P3GpuCtx, field: c_int, d_trace: *mut u32, h: usize, w: usize) -> i32;
    pub fn p3gpu_lde_coset_block_dev(ctx: *mut P3GpuCtx, field: c_int, d_coeffs: *const u32, h: usize, w: usize, added_bits: c_uint,
                                     shift: u32, coset: usize, d_out: *mut u32) -> i32;

    // Poseidon2 constants (drawn by Rust: Poseidon2::new / new_from_rng), Mmcs::commit
    pub fn p3gpu_poseidon2_set_constants(ctx: *mut P3GpuCtx, field: c_int, width: c_int, rc_initial: *const u32, rc_terminal: *const u32,
                                         rc_internal: *const u32, rounds_p: c_int) -> i32;
    pub fn p3gpu_merkle_total_digests(max_height: usize) -> usize;
    pub fn p3gpu_merkle_commit(ctx: *mut P3GpuCtx, field: c_int, hash: c_int, n_mats: usize, mats: *const *const u32, heights: *const usize,
                               widths: *const usize, layers: *mut u32, layer_lens: *mut usize, n_layers: *mut usize) -> i32;
    pub fn p3gpu_merkle_commit_dev(ctx: *mut P3GpuCtx, field: c_int, hash: c_int, n_mats: usize, d_mats: *const *const u32, heights: *const usize,
                                   widths: *const usize, d_layers: *mut u32, layer_lens: *mut usize, n_layers: *mut usize) -> i32;

    // FriFoldingStrategy::fold_matrix
    pub fn p3gpu_fri_fold(ctx: *mut P3GpuCtx, field: c_int, input: *const u32, rows: usize, log_arity: c_uint, beta: *const u32, out: *mut u32) -> i32;
    pub fn p3gpu_fri_fold_dev(ctx: *mut P3GpuCtx, field: c_int, d_in: *const u32, rows: usize, log_arity: c_uint, beta: *const u32, d_out: *mut u32) -> i32;
    pub fn p3gpu_ef_axpy_dev(ctx: *mut P3GpuCtx, field: c_int, d_acc: *mut u32, d_x: *const u32, n: usize, s: *const u32) -> i32;

    // Pcs::commit (host trace in, LDE + layers resident, cap out) and the device-resident variant
    pub fn p3gpu_pcs_commit(ctx: *mut P3GpuCtx, field: c_int, hash: c_int, h_evals: *const u32, h: usize, w: usize, log_blowup: c_uint,
                            cap_height: c_uint, d_lde: *mut u32, d_layers: *mut u32, layer_lens: *mut usize, n_layers: *mut usize,
                            h_cap: *mut u32, cap_len: *mut usize) -> i32;
    pub fn p3gpu_pcs_commit_dev(ctx: *mut P3GpuCtx, field: c_int, hash: c_int, d_evals: *const u32, h: usize, w: usize, log_blowup: c_uint,
                                d_lde: *mut u32, d_layers: *mut u32, layer_lens: *mut usize, n_layers: *mut usize) -> i32;

    // Pcs::open, pre-FRI part
    pub fn p3gpu_open_inv_denoms_dev(ctx: *mut P3GpuCtx, field: c_int, log_height: c_uint, z: *const u32, zinv: *const u32, d_inv_denoms: *mut u32,
                                     d_adjusted: *mut u32) -> i32;
    pub fn p3gpu_columnwise_dot_dev(ctx: *mut P3GpuCtx, field: c_int, d_mat: *const u32, h: usize, w: usize, d_vec_ef: *const u32, scale: *const u32,
                                    d_out: *mut u32) -> i32;
    pub fn p3gpu_rowwise_dot_dev(ctx: *mut P3GpuCtx, field: c_int, d_mat: *const u32, h: usize, w: usize, alpha: *const u32, d_out: *mut u32) -> i32;
    pub fn p3gpu_open_reduce_dev(ctx: *mut P3GpuCtx, field: c_int, d_ro: *mut u32, d_r: *const u32, d_inv_denoms: *const u32, h: usize,
                                 coeff: *const u32, yred: *const u32) -> i32;

    // query phase gathers
    pub fn p3gpu_gather_rows_dev(ctx: *mut P3GpuCtx, d_mat: *const u32, h: usize, w: usize, h_indices: *const u32, n: usize, index_shift: c_uint,
                                 d_out: *mut u32) -> i32;
    pub fn p3gpu_merkle_paths_dev(ctx: *mut P3GpuCtx, d_layers: *const u32, layer_lens: *const usize, n_layers: usize, path_len: usize,
                                  h_indices: *const u32, n: usize, index_shift: c_uint, d_out: *mut u32) -> i32;

    // multi-GPU (one process per GPU, CUDA IPC peer memory)
    pub fn p3gpu_ipc_export(ctx: *mut P3GpuCtx, dptr: *mut c_void, handle: *mut u8) -> i32;
    pub fn p3gpu_ipc_import(ctx: *mut P3GpuCtx, handle: *const u8, dptr: *mut *mut c_void) -> i32;
    pub fn p3gpu_ipc_close(ctx: *mut P3GpuCtx, dptr: *mut c_void) -> i32;
    pub fn p3gpu_peer_barrier_dev(ctx: *mut P3GpuCtx, grp: *const P3GpuPeerGroup, epoch: u32) -> i32;
    pub fn p3gpu_commit_sharded_dev(ctx: *mut P3GpuCtx, field: c_int, hash: c_int, grp: *const P3GpuPeerGroup, epoch: *mut u32,
                                    d_evals_local: *const u32, h: usize, col_starts: *const usize, log_blowup: c_uint,
                                    cap_height: c_uint, d_sub_layers: *mut u32, layer_lens: *mut usize, n_layers: *mut usize, h_cap: *mut u32,
                                    cap_len: *mut usize, phase_ms: *mut f32) -> i32;
    pub fn p3gpu_shard_chunk_bounds(w_local: usize, bounds: *mut usize, max_bounds: usize) -> usize;
    pub fn p3gpu_memset_dev(ctx: *mut P3GpuCtx, dptr: *mut c_void, value: c_int, bytes: usize) -> i32;
    pub fn p3gpu_peer_allgather_dev(ctx: *mut P3GpuCtx, grp: *const P3GpuPeerGroup, table_offset_bytes: usize, d_src: *const u32, words: usize) -> i32;
    pub fn p3gpu_coset_lde_batch_sharded_dev(ctx: *mut P3GpuCtx, field: c_int, grp: *const P3GpuPeerGroup, d_in: *const u32, h: usize,
                                             w_local: usize, added_bits: c_uint, shift: u32, w_total: usize, col_off: usize) -> i32;
    pub fn p3gpu_shard_col_segments(world: u32, col_starts: *const usize, rows: usize, segs: *mut usize, max_segs: usize, n_segs: *mut usize) -> i32;
    pub fn p3gpu_peer_exchange_dev(ctx: *mut P3GpuCtx, grp: *const P3GpuPeerGroup, epoch: *mut u32, bufs: *const *mut c_void, d_src: *const u32,
                                   words: usize) -> i32;
    pub fn p3gpu_p2air_quotient_sharded_dev(ctx: *mut P3GpuCtx, field: c_int, vector_len: c_int, grp: *const P3GpuPeerGroup, col_starts: *const usize,
                                            log_lde_height: c_uint, log_trace_height: c_uint, alpha: *const u32, d_quotient_slice: *mut u32) -> i32;
    pub fn p3gpu_blake3_air_quotient_sharded_dev(ctx: *mut P3GpuCtx, field: c_int, grp: *const P3GpuPeerGroup, col_starts: *const usize,
                                                 log_lde_height: c_uint, log_trace_height: c_uint, alpha: *const u32, d_quotient_slice: *mut u32) -> i32;
    pub fn p3gpu_sha256_air_quotient_sharded_dev(ctx: *mut P3GpuCtx, field: c_int, grp: *const P3GpuPeerGroup, col_starts: *const usize,
                                                 log_lde_height: c_uint, log_trace_height: c_uint, alpha: *const u32, d_quotient_slice: *mut u32) -> i32;
    pub fn p3gpu_p1air_quotient_sharded_dev(ctx: *mut P3GpuCtx, field: c_int, vector_len: c_int, grp: *const P3GpuPeerGroup, col_starts: *const usize,
                                            log_lde_height: c_uint, log_trace_height: c_uint, alpha: *const u32, d_quotient_slice: *mut u32) -> i32;
    pub fn p3gpu_air_quotient_sharded_dev(ctx: *mut P3GpuCtx, prog: *const P3GpuAirProgram, grp: *const P3GpuPeerGroup, col_starts: *const usize,
                                          d_periodic: *const u32, log_periodic_rows: c_uint, log_lde_height: c_uint, log_trace_height: c_uint,
                                          public_values: *const u32, alpha: *const u32, d_quotient_slice: *mut u32) -> i32;

    // streams, counters
    pub fn p3gpu_ctx_set_stream(ctx: *mut P3GpuCtx, cuda_stream: *mut c_void) -> i32;
    pub fn p3gpu_ctx_use_own_stream(ctx: *mut P3GpuCtx) -> i32;
    pub fn p3gpu_launch_count(ctx: *const P3GpuCtx) -> u64;

    // bare permutations, tree above given digests, bench-only commit phase with pre-drawn betas
    pub fn p3gpu_poseidon2_permute_dev(ctx: *mut P3GpuCtx, field: c_int, width: c_int, d_states: *mut u32, n: usize) -> i32;
    pub fn p3gpu_keccak_f_dev(ctx: *mut P3GpuCtx, d_states: *mut u64, n: usize) -> i32;
    pub fn p3gpu_merkle_from_digests_dev(ctx: *mut P3GpuCtx, field: c_int, hash: c_int, d_digests: *const u32, n: usize, d_layers: *mut u32,
                                         layer_lens: *mut usize, n_layers: *mut usize) -> i32;
    pub fn p3gpu_fri_commit_phase_dev(ctx: *mut P3GpuCtx, field: c_int, hash: c_int, d_vec: *mut u32, len: usize, log_blowup: c_uint,
                                      log_final_poly_len: c_uint, max_log_arity: c_uint, cap_height: c_uint, betas: *const u32, n_betas: usize,
                                      h_caps: *mut u32, cap_lens: *mut usize, log_arities: *mut c_uint, n_rounds: *mut usize, h_final: *mut u32) -> i32;

    // Poseidon2 AIR (poseidon2-air): trace generation and quotient values
    pub fn p3gpu_p2air_set_constants(ctx: *mut P3GpuCtx, field: c_int, beginning_full: *const u32, partial: *const u32, rounds_p: c_int,
                                     ending_full: *const u32) -> i32;
    pub fn p3gpu_p2air_columns(rounds_p: c_int) -> usize;
    pub fn p3gpu_p2air_field_columns(field: c_int, rounds_p: c_int) -> usize;
    pub fn p3gpu_p2air_generate_trace_dev(ctx: *mut P3GpuCtx, field: c_int, d_inputs: *const u32, n_perms: usize, d_trace: *mut u32) -> i32;
    pub fn p3gpu_p2air_quotient_dev(ctx: *mut P3GpuCtx, field: c_int, vector_len: c_int, d_lde: *const u32, log_lde_height: c_uint,
                                    log_trace_height: c_uint, alpha: *const u32, d_quotient: *mut u32) -> i32;
    pub fn p3gpu_p2air_generate_trace_cols_dev(ctx: *mut P3GpuCtx, field: c_int, vector_len: c_int, d_inputs: *const u32, n_perms: usize,
                                               col0: usize, col1: usize, d_out: *mut u32) -> i32;

    // Keccak-f AIR (keccak-air): trace generation and quotient values, P3GPU_KECCAK_AIR_COLS columns
    pub fn p3gpu_keccak_air_generate_trace_dev(ctx: *mut P3GpuCtx, field: c_int, d_inputs: *const u64, n_hashes: usize, d_trace: *mut u32) -> i32;
    pub fn p3gpu_keccak_air_quotient_dev(ctx: *mut P3GpuCtx, field: c_int, d_lde: *const u32, log_lde_height: c_uint, log_trace_height: c_uint,
                                         alpha: *const u32, d_quotient: *mut u32) -> i32;

    // Blake3 AIR (blake3-air): trace generation and quotient values, P3GPU_BLAKE3_AIR_COLS columns
    pub fn p3gpu_blake3_air_generate_trace_dev(ctx: *mut P3GpuCtx, field: c_int, d_inputs: *const u32, n_hashes: usize, d_trace: *mut u32) -> i32;
    pub fn p3gpu_blake3_air_quotient_dev(ctx: *mut P3GpuCtx, field: c_int, d_lde: *const u32, log_lde_height: c_uint, log_trace_height: c_uint,
                                         alpha: *const u32, d_quotient: *mut u32) -> i32;
    pub fn p3gpu_blake3_air_generate_trace_cols_dev(ctx: *mut P3GpuCtx, field: c_int, d_inputs: *const u32, n_hashes: usize, col0: usize,
                                                    col1: usize, d_out: *mut u32) -> i32;

    // SHA-256 AIR (sha256-air): trace generation and quotient values, P3GPU_SHA256_AIR_COLS columns
    pub fn p3gpu_sha256_air_generate_trace_dev(ctx: *mut P3GpuCtx, field: c_int, d_inputs: *const u32, n_hashes: usize, d_trace: *mut u32) -> i32;
    pub fn p3gpu_sha256_air_quotient_dev(ctx: *mut P3GpuCtx, field: c_int, d_lde: *const u32, log_lde_height: c_uint, log_trace_height: c_uint,
                                         alpha: *const u32, d_quotient: *mut u32) -> i32;
    pub fn p3gpu_sha256_air_generate_trace_cols_dev(ctx: *mut P3GpuCtx, field: c_int, d_inputs: *const u32, n_hashes: usize, col0: usize,
                                                    col1: usize, d_out: *mut u32) -> i32;

    // Poseidon1 AIR (poseidon1-air, width 16): per-context constants (Poseidon1Constants::to_optimized's output, Montgomery words),
    // trace generation and quotient values
    pub fn p3gpu_p1air_set_constants(ctx: *mut P3GpuCtx, field: c_int, initial_full: *const u32, terminal_full: *const u32,
                                     mds_circ_col: *const u32, first_round_constants: *const u32, m_i: *const u32, partial_rc: *const u32,
                                     sparse_first_row: *const u32, v: *const u32, rounds_p: c_int) -> i32;
    pub fn p3gpu_p1air_columns(field: c_int, rounds_p: c_int) -> usize;
    pub fn p3gpu_p1air_generate_trace_dev(ctx: *mut P3GpuCtx, field: c_int, d_inputs: *const u32, n_perms: usize, d_trace: *mut u32) -> i32;
    pub fn p3gpu_p1air_quotient_dev(ctx: *mut P3GpuCtx, field: c_int, vector_len: c_int, d_lde: *const u32, log_lde_height: c_uint,
                                    log_trace_height: c_uint, alpha: *const u32, d_quotient: *mut u32) -> i32;
    pub fn p3gpu_p1air_generate_trace_cols_dev(ctx: *mut P3GpuCtx, field: c_int, vector_len: c_int, d_inputs: *const u32, n_perms: usize,
                                               col0: usize, col1: usize, d_out: *mut u32) -> i32;

    // any AIR as a constraint program (symbolic expression DAG -> register program -> quotient kernel)
    pub fn p3gpu_air_program_create(ctx: *mut P3GpuCtx, field: c_int, nodes: *const P3GpuAirNode, n_nodes: usize, constraints: *const u32,
                                    n_constraints: usize, width: u32, n_public: u32, out: *mut *mut P3GpuAirProgram) -> i32;
    pub fn p3gpu_air_program_create_layout(ctx: *mut P3GpuCtx, field: c_int, nodes: *const P3GpuAirNode, n_nodes: usize,
                                           constraints: *const u32, n_constraints: usize, layout: *const P3GpuAirLayout,
                                           out: *mut *mut P3GpuAirProgram) -> i32;
    pub fn p3gpu_air_program_destroy(prog: *mut P3GpuAirProgram);
    pub fn p3gpu_air_program_info(prog: *const P3GpuAirProgram, n_instructions: *mut usize, n_slots: *mut usize, n_constraints: *mut usize) -> i32;
    pub fn p3gpu_air_quotient_dev(ctx: *mut P3GpuCtx, prog: *const P3GpuAirProgram, d_lde: *const u32, log_lde_height: c_uint,
                                  log_quotient_size: c_uint, log_trace_height: c_uint, public_values: *const u32, alpha: *const u32,
                                  d_quotient: *mut u32) -> i32;
    pub fn p3gpu_air_quotient_layout_dev(ctx: *mut P3GpuCtx, prog: *const P3GpuAirProgram, d_lde: *const u32, log_lde_height: c_uint,
                                         d_pre_lde: *const u32, log_pre_lde_height: c_uint, d_periodic: *const u32,
                                         log_periodic_rows: c_uint, log_quotient_size: c_uint, log_trace_height: c_uint,
                                         public_values: *const u32, alpha: *const u32, d_quotient: *mut u32) -> i32;

    // the debug constraint check of any AIR over the trace domain (pass 1: per-row failure counts; pass 2: the listed rows' failures)
    pub fn p3gpu_air_check_program_create(ctx: *mut P3GpuCtx, field: c_int, nodes: *const P3GpuAirNode, n_nodes: usize,
                                          constraints: *const u32, n_constraints: usize, layout: *const P3GpuAirLayout,
                                          out: *mut *mut P3GpuAirProgram) -> i32;
    pub fn p3gpu_air_check_dev(ctx: *mut P3GpuCtx, prog: *const P3GpuAirProgram, d_trace: *const u32, height: usize, d_preprocessed: *const u32,
                               d_periodic: *const u32, periodic_rows: usize, public_values: *const u32, d_counts: *mut u32) -> i32;
    pub fn p3gpu_air_check_rows_dev(ctx: *mut P3GpuCtx, prog: *const P3GpuAirProgram, d_trace: *const u32, height: usize,
                                    d_preprocessed: *const u32, d_periodic: *const u32, periodic_rows: usize, public_values: *const u32,
                                    d_rows: *const u32, n_rows: usize, d_offsets: *const u64, d_failed: *mut u32) -> i32;

    // DuplexChallenger with device-resident state
    pub fn p3gpu_challenger_new(ctx: *mut P3GpuCtx, field: c_int, width: c_int, rate: c_int, out: *mut *mut P3GpuChallenger) -> i32;
    pub fn p3gpu_challenger_free(ctx: *mut P3GpuCtx, ch: *mut P3GpuChallenger);
    pub fn p3gpu_challenger_clone(ctx: *mut P3GpuCtx, src: *const P3GpuChallenger, out: *mut *mut P3GpuChallenger) -> i32;
    pub fn p3gpu_challenger_observe_dev(ctx: *mut P3GpuCtx, ch: *mut P3GpuChallenger, d_values: *const u32, n: usize) -> i32;
    pub fn p3gpu_challenger_observe(ctx: *mut P3GpuCtx, ch: *mut P3GpuChallenger, h_values: *const u32, n: usize) -> i32;
    pub fn p3gpu_challenger_sample(ctx: *mut P3GpuCtx, ch: *mut P3GpuChallenger, h_out: *mut u32, n: usize) -> i32;
    pub fn p3gpu_challenger_grind(ctx: *mut P3GpuCtx, ch: *mut P3GpuChallenger, bits: c_uint, witness: *mut u32) -> i32;
    pub fn p3gpu_challenger_new_keccak256(ctx: *mut P3GpuCtx, field: c_int, out: *mut *mut P3GpuChallenger) -> i32;
    pub fn p3gpu_challenger_new_sha256(ctx: *mut P3GpuCtx, field: c_int, out: *mut *mut P3GpuChallenger) -> i32;
    pub fn p3gpu_challenger_observe_digest(ctx: *mut P3GpuCtx, ch: *mut P3GpuChallenger, h_words: *const u32, n: usize) -> i32;
    pub fn p3gpu_challenger_sample_bits(ctx: *mut P3GpuCtx, ch: *mut P3GpuChallenger, bits: c_uint, n: usize, h_out: *mut u32) -> i32;
}

/// The reference's prover-side trait methods have no `Result`: shape violations panic (`log2_strict_usize`,
/// `mmcs/batch.rs:50-54`).  The shim keeps that behaviour.
pub fn check(rc: i32) {
    if rc != 0 {
        let msg = unsafe { core::ffi::CStr::from_ptr(p3gpu_last_error()) }.to_string_lossy();
        panic!("p3gpu error {rc}: {msg}");
    }
}
