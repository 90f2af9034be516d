"""ctypes binding of libp3gpu.so (include/p3gpu.h).  There is NO fallback: if the CUDA library is missing or no
device is present, importing callers get a hard error."""
from __future__ import annotations

import ctypes as C
import os
import pathlib

_HERE = pathlib.Path(__file__).resolve().parent
# P3GPU_LIB selects another build of the same library (e.g. the -DP3GPU_NTT_PROFILE instrumented one); never a fallback
LIB_PATH = pathlib.Path(os.environ["P3GPU_LIB"]) if os.environ.get("P3GPU_LIB") else _HERE / "libp3gpu.so"

BABY_BEAR, KOALA_BEAR = 0, 1
EOK, EINVAL, EUNSUPPORTED, ECUDA, ENOMEM, ESTATE = 0, -1, -2, -3, -4, -5
DFT, IDFT, COSET_DFT, COSET_IDFT = 0, 1, 2, 3
HASH_POSEIDON2_W16, HASH_POSEIDON2_W24, HASH_KECCAK, HASH_SHA256, HASH_SHA256_COMPRESS = 0, 1, 2, 3, 4
KECCAK_AIR_COLS = 2633                       # P3GPU_KECCAK_AIR_COLS
BLAKE3_AIR_COLS = 9168                       # P3GPU_BLAKE3_AIR_COLS
SHA256_AIR_COLS = 7728                       # P3GPU_SHA256_AIR_COLS

EXPORTS = [
    "p3gpu_ctx_create", "p3gpu_ctx_destroy", "p3gpu_ctx_set_stream", "p3gpu_ctx_use_own_stream", "p3gpu_ctx_sync", "p3gpu_last_error",
    "p3gpu_launch_count", "p3gpu_malloc", "p3gpu_free", "p3gpu_memcpy_h2d", "p3gpu_memcpy_d2h",
    "p3gpu_host_register", "p3gpu_host_unregister",
    "p3gpu_dft_batch_dev", "p3gpu_dft_batch", "p3gpu_coset_lde_batch_dev", "p3gpu_coset_lde_batch",
    "p3gpu_poseidon2_set_constants", "p3gpu_poseidon2_permute_dev", "p3gpu_keccak_f_dev",
    "p3gpu_merkle_total_digests", "p3gpu_merkle_commit_dev", "p3gpu_merkle_commit", "p3gpu_merkle_from_digests_dev",
    "p3gpu_fri_fold_dev", "p3gpu_fri_fold", "p3gpu_ef_axpy_dev", "p3gpu_fri_commit_phase_dev", "p3gpu_pcs_commit_dev",
    "p3gpu_open_inv_denoms_dev", "p3gpu_columnwise_dot_dev", "p3gpu_rowwise_dot_dev", "p3gpu_open_reduce_dev",
    "p3gpu_pcs_commit", "p3gpu_p2air_set_constants", "p3gpu_p2air_columns", "p3gpu_p2air_field_columns", "p3gpu_p2air_generate_trace_dev", "p3gpu_p2air_quotient_dev",
    "p3gpu_challenger_new", "p3gpu_challenger_free", "p3gpu_challenger_clone", "p3gpu_challenger_observe_dev", "p3gpu_challenger_observe",
    "p3gpu_challenger_sample", "p3gpu_challenger_grind", "p3gpu_gather_rows_dev", "p3gpu_merkle_paths_dev",
    "p3gpu_ipc_export", "p3gpu_ipc_import", "p3gpu_ipc_close", "p3gpu_memset_dev", "p3gpu_peer_barrier_dev",
    "p3gpu_peer_allgather_dev", "p3gpu_coset_lde_batch_sharded_dev", "p3gpu_commit_sharded_dev", "p3gpu_shard_chunk_bounds",
    "p3gpu_p2air_generate_trace_cols_dev", "p3gpu_shard_col_segments", "p3gpu_peer_exchange_dev", "p3gpu_p2air_quotient_sharded_dev",
    "p3gpu_air_program_create", "p3gpu_air_program_destroy", "p3gpu_air_program_info", "p3gpu_air_quotient_dev",
    "p3gpu_air_program_create_layout", "p3gpu_air_quotient_layout_dev",
    "p3gpu_air_check_program_create", "p3gpu_air_check_dev", "p3gpu_air_check_rows_dev",
    "p3gpu_challenger_new_keccak256", "p3gpu_challenger_observe_digest", "p3gpu_challenger_sample_bits",
    "p3gpu_challenger_new_sha256",
    "p3gpu_keccak_air_generate_trace_dev", "p3gpu_keccak_air_quotient_dev",
    "p3gpu_blake3_air_generate_trace_dev", "p3gpu_blake3_air_quotient_dev",
    "p3gpu_sha256_air_generate_trace_dev", "p3gpu_sha256_air_quotient_dev",
    "p3gpu_p1air_set_constants", "p3gpu_p1air_columns", "p3gpu_p1air_generate_trace_dev", "p3gpu_p1air_quotient_dev",
    "p3gpu_blake3_air_generate_trace_cols_dev", "p3gpu_sha256_air_generate_trace_cols_dev", "p3gpu_p1air_generate_trace_cols_dev",
    "p3gpu_blake3_air_quotient_sharded_dev", "p3gpu_sha256_air_quotient_sharded_dev", "p3gpu_p1air_quotient_sharded_dev",
    "p3gpu_air_quotient_sharded_dev",
    "p3gpu_lde_coefficients_dev", "p3gpu_lde_coset_block_dev",
]

PEER_CTRL_BYTES, PEER_CTRL_USER = 65536, 256


class PeerGroupStruct(C.Structure):
    """p3gpu_peer_group (include/p3gpu.h)."""
    _fields_ = [("world", C.c_uint32), ("rank", C.c_uint32), ("ctrl", C.c_void_p * 16), ("rows", C.c_void_p * 16),
                ("timeout_s", C.c_double)]


class P3GpuError(RuntimeError):
    """A non-zero return code of the library; `code` is the P3GPU_E* value (0 for errors raised before any call)."""

    def __init__(self, msg, code=0):
        super().__init__(msg)
        self.code = code


_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise P3GpuError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                         "(plonky3_b200/csrc/build.sh).  There is no CPU fallback.")
    L = C.CDLL(str(LIB_PATH))
    vp, sz, u32, i32, ci, cu = C.c_void_p, C.c_size_t, C.c_uint32, C.c_int32, C.c_int, C.c_uint
    sig = {
        "p3gpu_ctx_create": (i32, [ci, C.POINTER(vp)]),
        "p3gpu_ctx_destroy": (None, [vp]),
        "p3gpu_ctx_set_stream": (i32, [vp, vp]),
        "p3gpu_ctx_use_own_stream": (i32, [vp]),
        "p3gpu_ctx_sync": (i32, [vp]),
        "p3gpu_last_error": (C.c_char_p, []),
        "p3gpu_launch_count": (C.c_uint64, [vp]),
        "p3gpu_malloc": (i32, [vp, sz, C.POINTER(vp)]),
        "p3gpu_free": (i32, [vp, vp]),
        "p3gpu_memcpy_h2d": (i32, [vp, vp, vp, sz]),
        "p3gpu_memcpy_d2h": (i32, [vp, vp, vp, sz]),
        "p3gpu_host_register": (i32, [vp, sz]),
        "p3gpu_host_unregister": (i32, [vp]),
        "p3gpu_dft_batch_dev": (i32, [vp, ci, ci, vp, vp, sz, sz, u32]),
        "p3gpu_dft_batch": (i32, [vp, ci, ci, vp, sz, sz, u32]),
        "p3gpu_coset_lde_batch_dev": (i32, [vp, ci, vp, sz, sz, cu, u32, vp, ci]),
        "p3gpu_coset_lde_batch": (i32, [vp, ci, vp, sz, sz, cu, u32, vp, ci]),
        "p3gpu_poseidon2_set_constants": (i32, [vp, ci, ci, vp, vp, vp, ci]),
        "p3gpu_poseidon2_permute_dev": (i32, [vp, ci, ci, vp, sz]),
        "p3gpu_keccak_f_dev": (i32, [vp, vp, sz]),
        "p3gpu_merkle_total_digests": (sz, [sz]),
        "p3gpu_merkle_commit_dev": (i32, [vp, ci, ci, sz, vp, vp, vp, vp, vp, vp]),
        "p3gpu_merkle_commit": (i32, [vp, ci, ci, sz, vp, vp, vp, vp, vp, vp]),
        "p3gpu_merkle_from_digests_dev": (i32, [vp, ci, ci, vp, sz, vp, vp, vp]),
        "p3gpu_fri_fold_dev": (i32, [vp, ci, vp, sz, cu, vp, vp]),
        "p3gpu_fri_fold": (i32, [vp, ci, vp, sz, cu, vp, vp]),
        "p3gpu_ef_axpy_dev": (i32, [vp, ci, vp, vp, sz, vp]),
        "p3gpu_fri_commit_phase_dev": (i32, [vp, ci, ci, vp, sz, cu, cu, cu, cu, vp, sz, vp, vp, vp, vp, vp]),
        "p3gpu_open_inv_denoms_dev": (i32, [vp, ci, cu, vp, vp, vp, vp]),
        "p3gpu_columnwise_dot_dev": (i32, [vp, ci, vp, sz, sz, vp, vp, vp]),
        "p3gpu_rowwise_dot_dev": (i32, [vp, ci, vp, sz, sz, vp, vp]),
        "p3gpu_open_reduce_dev": (i32, [vp, ci, vp, vp, vp, sz, vp, vp]),
        "p3gpu_pcs_commit_dev": (i32, [vp, ci, ci, vp, sz, sz, cu, vp, vp, vp, vp]),
        "p3gpu_pcs_commit": (i32, [vp, ci, ci, vp, sz, sz, cu, cu, vp, vp, vp, vp, vp, vp]),
        "p3gpu_p2air_set_constants": (i32, [vp, ci, vp, vp, ci, vp]),
        "p3gpu_p2air_columns": (sz, [ci]),
        "p3gpu_p2air_field_columns": (sz, [ci, ci]),
        "p3gpu_p2air_generate_trace_dev": (i32, [vp, ci, vp, sz, vp]),
        "p3gpu_p2air_quotient_dev": (i32, [vp, ci, ci, vp, cu, cu, vp, vp]),
        "p3gpu_challenger_new": (i32, [vp, ci, ci, ci, C.POINTER(vp)]),
        "p3gpu_challenger_free": (None, [vp, vp]),
        "p3gpu_challenger_clone": (i32, [vp, vp, C.POINTER(vp)]),
        "p3gpu_challenger_observe_dev": (i32, [vp, vp, vp, sz]),
        "p3gpu_challenger_observe": (i32, [vp, vp, vp, sz]),
        "p3gpu_challenger_sample": (i32, [vp, vp, vp, sz]),
        "p3gpu_challenger_grind": (i32, [vp, vp, cu, vp]),
        "p3gpu_gather_rows_dev": (i32, [vp, vp, sz, sz, vp, sz, cu, vp]),
        "p3gpu_merkle_paths_dev": (i32, [vp, vp, vp, sz, sz, vp, sz, cu, vp]),
        "p3gpu_ipc_export": (i32, [vp, vp, vp]),
        "p3gpu_ipc_import": (i32, [vp, vp, C.POINTER(vp)]),
        "p3gpu_ipc_close": (i32, [vp, vp]),
        "p3gpu_memset_dev": (i32, [vp, vp, ci, sz]),
        "p3gpu_peer_barrier_dev": (i32, [vp, vp, u32]),
        "p3gpu_peer_allgather_dev": (i32, [vp, vp, sz, vp, sz]),
        "p3gpu_coset_lde_batch_sharded_dev": (i32, [vp, ci, vp, vp, sz, sz, cu, u32, sz, sz]),
        "p3gpu_commit_sharded_dev": (i32, [vp, ci, ci, vp, vp, vp, sz, vp, cu, cu, vp, vp, vp, vp, vp, vp]),
        "p3gpu_shard_chunk_bounds": (sz, [sz, vp, sz]),
        "p3gpu_p2air_generate_trace_cols_dev": (i32, [vp, ci, ci, vp, sz, sz, sz, vp]),
        "p3gpu_shard_col_segments": (i32, [u32, vp, sz, vp, sz, vp]),
        "p3gpu_peer_exchange_dev": (i32, [vp, vp, vp, vp, vp, sz]),
        "p3gpu_p2air_quotient_sharded_dev": (i32, [vp, ci, ci, vp, vp, cu, cu, vp, vp]),
        "p3gpu_air_program_create": (i32, [vp, ci, vp, sz, vp, sz, u32, u32, C.POINTER(vp)]),
        "p3gpu_air_program_destroy": (None, [vp]),
        "p3gpu_air_program_info": (i32, [vp, C.POINTER(sz), C.POINTER(sz), C.POINTER(sz)]),
        "p3gpu_air_quotient_dev": (i32, [vp, vp, vp, cu, cu, cu, vp, vp, vp]),
        "p3gpu_air_program_create_layout": (i32, [vp, ci, vp, sz, vp, sz, vp, C.POINTER(vp)]),
        "p3gpu_air_quotient_layout_dev": (i32, [vp, vp, vp, cu, vp, cu, vp, cu, cu, cu, vp, vp, vp]),
        "p3gpu_air_check_program_create": (i32, [vp, ci, vp, sz, vp, sz, vp, C.POINTER(vp)]),
        "p3gpu_air_check_dev": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp]),
        "p3gpu_air_check_rows_dev": (i32, [vp, vp, vp, sz, vp, vp, sz, vp, vp, sz, vp, vp]),
        "p3gpu_challenger_new_keccak256": (i32, [vp, ci, C.POINTER(vp)]),
        "p3gpu_challenger_new_sha256": (i32, [vp, ci, C.POINTER(vp)]),
        "p3gpu_challenger_observe_digest": (i32, [vp, vp, vp, sz]),
        "p3gpu_challenger_sample_bits": (i32, [vp, vp, cu, sz, vp]),
        "p3gpu_keccak_air_generate_trace_dev": (i32, [vp, ci, vp, sz, vp]),
        "p3gpu_keccak_air_quotient_dev": (i32, [vp, ci, vp, cu, cu, vp, vp]),
        "p3gpu_blake3_air_generate_trace_dev": (i32, [vp, ci, vp, sz, vp]),
        "p3gpu_blake3_air_quotient_dev": (i32, [vp, ci, vp, cu, cu, vp, vp]),
        "p3gpu_sha256_air_generate_trace_dev": (i32, [vp, ci, vp, sz, vp]),
        "p3gpu_sha256_air_quotient_dev": (i32, [vp, ci, vp, cu, cu, vp, vp]),
        "p3gpu_p1air_set_constants": (i32, [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp, ci]),
        "p3gpu_p1air_columns": (sz, [ci, ci]),
        "p3gpu_p1air_generate_trace_dev": (i32, [vp, ci, vp, sz, vp]),
        "p3gpu_p1air_quotient_dev": (i32, [vp, ci, ci, vp, cu, cu, vp, vp]),
        "p3gpu_blake3_air_generate_trace_cols_dev": (i32, [vp, ci, vp, sz, sz, sz, vp]),
        "p3gpu_sha256_air_generate_trace_cols_dev": (i32, [vp, ci, vp, sz, sz, sz, vp]),
        "p3gpu_p1air_generate_trace_cols_dev": (i32, [vp, ci, ci, vp, sz, sz, sz, vp]),
        "p3gpu_blake3_air_quotient_sharded_dev": (i32, [vp, ci, vp, vp, cu, cu, vp, vp]),
        "p3gpu_sha256_air_quotient_sharded_dev": (i32, [vp, ci, vp, vp, cu, cu, vp, vp]),
        "p3gpu_p1air_quotient_sharded_dev": (i32, [vp, ci, ci, vp, vp, cu, cu, vp, vp]),
        "p3gpu_air_quotient_sharded_dev": (i32, [vp, vp, vp, vp, vp, cu, cu, cu, vp, vp, vp]),
        "p3gpu_lde_coefficients_dev": (i32, [vp, ci, vp, sz, sz]),
        "p3gpu_lde_coset_block_dev": (i32, [vp, ci, vp, sz, sz, cu, u32, sz, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        raise P3GpuError(f"libp3gpu error {rc}: {load().p3gpu_last_error().decode()}", rc)
