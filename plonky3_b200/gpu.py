"""Thin object wrapper over the libp3gpu C ABI (include/p3gpu.h).

A matrix is either a numpy uint32 array (HOST: the call goes through the host-pointer entry points and includes
the PCIe copies) or a torch CUDA int32 tensor (DEVICE: the `_dev` entry points run on torch's current stream and
the result is a new CUDA tensor).  PyTorch is used only for device memory and streams.
All values are Montgomery-form u32 (MontyField31.value, monty-31/src/monty_31.rs:34-44).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import check


def _is_torch(x):
    return type(x).__module__.startswith("torch")


class Gpu:
    """One libp3gpu context bound to one CUDA device."""

    def __init__(self, device: int = 0):
        self.L = _lib.load()
        h = C.c_void_p()
        check(self.L.p3gpu_ctx_create(device, C.byref(h)))
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.L.p3gpu_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ plumbing
    def _use_torch_stream(self):
        import torch
        check(self.L.p3gpu_ctx_set_stream(self.h, C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))

    def _empty(self, shape):
        import torch
        return torch.empty(shape, dtype=torch.int32, device=f"cuda:{self.device}")

    @staticmethod
    def _np(a):
        a = np.ascontiguousarray(a, dtype=np.uint32)
        if a.ndim == 1:
            a = a.reshape(-1, 1)
        return a

    @staticmethod
    def _dev(t):
        import torch
        assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous(), "device matrices are contiguous CUDA int32 tensors"
        return t

    def sync(self):
        check(self.L.p3gpu_ctx_sync(self.h))

    @property
    def launches(self) -> int:
        return int(self.L.p3gpu_launch_count(self.h))

    # ------------------------------------------------------------------ TwoAdicSubgroupDft
    def dft_batch(self, field, kind, mat, shift=0):
        if _is_torch(mat):
            m = self._dev(mat); self._use_torch_stream()
            out = self._empty(tuple(m.shape))
            check(self.L.p3gpu_dft_batch_dev(self.h, field, kind, m.data_ptr(), out.data_ptr(), m.shape[0], m.shape[1], shift))
            return out
        m = self._np(mat).copy()
        check(self.L.p3gpu_dft_batch(self.h, field, kind, m.ctypes.data, m.shape[0], m.shape[1], shift))
        return m

    def coset_lde_batch(self, field, mat, added_bits, shift, bitrev_rows=True):
        if _is_torch(mat):
            m = self._dev(mat); self._use_torch_stream()
            out = self._empty((m.shape[0] << added_bits, m.shape[1]))
            check(self.L.p3gpu_coset_lde_batch_dev(self.h, field, m.data_ptr(), m.shape[0], m.shape[1], added_bits, shift,
                                                   out.data_ptr(), int(bitrev_rows)))
            return out
        m = self._np(mat)
        out = np.empty((m.shape[0] << added_bits, m.shape[1]), dtype=np.uint32)
        check(self.L.p3gpu_coset_lde_batch(self.h, field, m.ctypes.data, m.shape[0], m.shape[1], added_bits, shift,
                                           out.ctypes.data, int(bitrev_rows)))
        return out

    def lde_coefficients(self, field, trace_dev):
        """p3gpu_lde_coefficients_dev: the device trace (h, w) becomes, in place, the coefficient form `lde_coset_block` reads.
        Returns the same tensor; its trace values are gone."""
        m = self._dev(trace_dev); self._use_torch_stream()
        check(self.L.p3gpu_lde_coefficients_dev(self.h, field, m.data_ptr(), m.shape[0], m.shape[1]))
        return m

    def lde_coset_block(self, field, coeffs_dev, added_bits, shift, coset, out=None):
        """p3gpu_lde_coset_block_dev: rows [coset h, (coset + 1) h) of coset_lde_batch(trace, added_bits, shift) from the trace's
        `lde_coefficients`, into `out` (a contiguous (h, w) CUDA int32 tensor, new if None).  Returns it."""
        m = self._dev(coeffs_dev); self._use_torch_stream()
        o = self._empty(tuple(m.shape)) if out is None else self._dev(out)
        assert tuple(o.shape) == tuple(m.shape), "the coset block has the trace's shape"
        check(self.L.p3gpu_lde_coset_block_dev(self.h, field, m.data_ptr(), m.shape[0], m.shape[1], added_bits, shift, coset, o.data_ptr()))
        return o

    # ------------------------------------------------------------------ hashing
    def poseidon2_set_constants(self, field, width, rc_initial, rc_terminal, rc_internal):
        a = np.ascontiguousarray(rc_initial, dtype=np.uint32).ravel()
        b = np.ascontiguousarray(rc_terminal, dtype=np.uint32).ravel()
        c = np.ascontiguousarray(rc_internal, dtype=np.uint32).ravel()
        if a.size != 4 * width or b.size != 4 * width:
            raise ValueError("external constants must be 4 x width")
        check(self.L.p3gpu_poseidon2_set_constants(self.h, field, width, a.ctypes.data, b.ctypes.data, c.ctypes.data, c.size))

    def poseidon2_permute(self, field, width, states):
        """states: (n, width) numpy uint32 or CUDA tensor; returns the permuted states."""
        import torch
        if _is_torch(states):
            s = self._dev(states).clone()
        else:
            s = torch.from_numpy(np.ascontiguousarray(states, dtype=np.uint32).view(np.int32)).to(f"cuda:{self.device}")
        self._use_torch_stream()
        check(self.L.p3gpu_poseidon2_permute_dev(self.h, field, width, s.data_ptr(), s.shape[0]))
        return s if _is_torch(states) else s.cpu().numpy().view(np.uint32)

    def keccak_f(self, states):
        import torch
        s = torch.from_numpy(np.ascontiguousarray(states, dtype=np.uint64).view(np.int64)).to(f"cuda:{self.device}")
        self._use_torch_stream()
        check(self.L.p3gpu_keccak_f_dev(self.h, s.data_ptr(), s.shape[0]))
        return s.cpu().numpy().view(np.uint64)

    def merkle_total_digests(self, max_height):
        return int(self.L.p3gpu_merkle_total_digests(max_height))

    def merkle_commit(self, field, hash_kind, mats):
        """MerkleTree::new.  Returns the list of digest layers ((len, 8) arrays/tensors, layer 0 = leaves)."""
        n = len(mats)
        if n == 0:
            raise _lib.P3GpuError("No matrices given?")
        dev = _is_torch(mats[0])
        ms = [self._dev(m) if dev else self._np(m) for m in mats]
        hts = (C.c_size_t * n)(*[int(m.shape[0]) for m in ms])
        wds = (C.c_size_t * n)(*[int(m.shape[1]) for m in ms])
        tot = self.merkle_total_digests(max(int(m.shape[0]) for m in ms))
        lens = (C.c_size_t * 65)()
        nl = C.c_size_t()
        if dev:
            self._use_torch_stream()
            ptrs = (C.c_void_p * n)(*[m.data_ptr() for m in ms])
            out = self._empty((max(tot, 1), 8))
            check(self.L.p3gpu_merkle_commit_dev(self.h, field, hash_kind, n, ptrs, hts, wds, out.data_ptr(), lens, C.byref(nl)))
        else:
            ptrs = (C.c_void_p * n)(*[m.ctypes.data for m in ms])
            out = np.zeros((max(tot, 1), 8), dtype=np.uint32)
            check(self.L.p3gpu_merkle_commit(self.h, field, hash_kind, n, ptrs, hts, wds, out.ctypes.data, lens, C.byref(nl)))
        layers, off = [], 0
        for k in range(nl.value):
            layers.append(out[off:off + lens[k]]); off += lens[k]
        return layers

    def merkle_from_digests(self, field, hash_kind, digests_dev):
        """Layers above an existing digest layer (CUDA tensor (n, 8)).  Returns [padded input layer, ..., root]."""
        d = self._dev(digests_dev); self._use_torch_stream()
        n = int(d.shape[0])
        out = self._empty((self.merkle_total_digests(n), 8))
        lens = (C.c_size_t * 65)(); nl = C.c_size_t()
        check(self.L.p3gpu_merkle_from_digests_dev(self.h, field, hash_kind, d.data_ptr(), n, out.data_ptr(), lens, C.byref(nl)))
        layers, off = [], 0
        for k in range(nl.value):
            layers.append(out[off:off + lens[k]]); off += lens[k]
        return layers

    # ------------------------------------------------------------------ FRI
    def fri_fold(self, field, vec_ef, log_arity, beta):
        b = np.ascontiguousarray(beta, dtype=np.uint32)
        assert b.size == 4
        if _is_torch(vec_ef):
            v = self._dev(vec_ef); self._use_torch_stream()
            rows = (v.numel() // 4) >> log_arity
            out = self._empty((rows, 4))
            check(self.L.p3gpu_fri_fold_dev(self.h, field, v.data_ptr(), rows, log_arity, b.ctypes.data, out.data_ptr()))
            return out
        v = np.ascontiguousarray(vec_ef, dtype=np.uint32)
        rows = (v.size // 4) >> log_arity
        out = np.empty((rows, 4), dtype=np.uint32)
        check(self.L.p3gpu_fri_fold(self.h, field, v.ctypes.data, rows, log_arity, b.ctypes.data, out.ctypes.data))
        return out

    def ef_axpy(self, field, acc_dev, x_dev, s):
        """acc += s * x over EF4, in place on the device (commit_phase roll-in, prover.rs:258-265)."""
        a, x = self._dev(acc_dev), self._dev(x_dev); self._use_torch_stream()
        sv = np.ascontiguousarray(s, dtype=np.uint32)
        assert a.numel() == x.numel() and sv.size == 4
        check(self.L.p3gpu_ef_axpy_dev(self.h, field, a.data_ptr(), x.data_ptr(), a.numel() // 4, sv.ctypes.data))
        return a

    def fri_commit_phase(self, field, hash_kind, vec_ef_dev, log_blowup, log_final_poly_len, max_log_arity, cap_height, betas):
        """All commit-phase rounds on the device with caller-supplied betas.  vec_ef_dev (CUDA, consumed).
        Returns (caps: list of (n,8) arrays, log_arities, final (len,4) array)."""
        v = self._dev(vec_ef_dev); self._use_torch_stream()
        length = v.numel() // 4
        b = np.ascontiguousarray(betas, dtype=np.uint32).reshape(-1, 4)
        caps = np.zeros((64 * (1 << cap_height), 8), dtype=np.uint32)
        cap_lens = (C.c_size_t * 64)(); las = (C.c_uint * 64)(); nr = C.c_size_t()
        final = np.zeros((1 << (log_blowup + log_final_poly_len), 4), dtype=np.uint32)
        check(self.L.p3gpu_fri_commit_phase_dev(self.h, field, hash_kind, v.data_ptr(), length, log_blowup, log_final_poly_len,
                                                max_log_arity, cap_height, b.ctypes.data, b.shape[0], caps.ctypes.data, cap_lens, las,
                                                C.byref(nr), final.ctypes.data))
        out, off = [], 0
        for k in range(nr.value):
            out.append(caps[off:off + cap_lens[k]].copy()); off += cap_lens[k]
        return out, [int(las[k]) for k in range(nr.value)], final

    # ------------------------------------------------------------------ Pcs::open (pre-FRI part)
    @staticmethod
    def _ef(a):
        a = np.ascontiguousarray(a, dtype=np.uint32)
        assert a.size == 4
        return a

    def open_inv_denoms(self, field, log_height, z, zinv=None):
        """(inv_denoms, adjusted or None): CUDA (2^log_height, 4) tensors, bit-reversed coset order."""
        self._use_torch_stream()
        zz = self._ef(z)
        inv = self._empty((1 << log_height, 4))
        adj = self._empty((1 << log_height, 4)) if zinv is not None else None
        zi = self._ef(zinv) if zinv is not None else None
        check(self.L.p3gpu_open_inv_denoms_dev(self.h, field, log_height, zz.ctypes.data, zi.ctypes.data if zi is not None else None,
                                               inv.data_ptr(), adj.data_ptr() if adj is not None else None))
        return inv, adj

    def columnwise_dot(self, field, mat, vec_ef, scale=None):
        m, v = self._dev(mat), self._dev(vec_ef); self._use_torch_stream()
        assert v.shape[0] >= m.shape[0]
        out = self._empty((int(m.shape[1]), 4))
        sc = self._ef(scale) if scale is not None else None
        check(self.L.p3gpu_columnwise_dot_dev(self.h, field, m.data_ptr(), m.shape[0], m.shape[1], v.data_ptr(),
                                              sc.ctypes.data if sc is not None else None, out.data_ptr()))
        return out

    def rowwise_dot(self, field, mat, alpha):
        m = self._dev(mat); self._use_torch_stream()
        out = self._empty((int(m.shape[0]), 4))
        a = self._ef(alpha)
        check(self.L.p3gpu_rowwise_dot_dev(self.h, field, m.data_ptr(), m.shape[0], m.shape[1], a.ctypes.data, out.data_ptr()))
        return out

    def open_reduce(self, field, ro, r, inv_denoms, coeff, yred):
        a, b, c = self._dev(ro), self._dev(r), self._dev(inv_denoms); self._use_torch_stream()
        h = int(a.shape[0])
        assert b.shape[0] == h and c.shape[0] >= h
        check(self.L.p3gpu_open_reduce_dev(self.h, field, a.data_ptr(), b.data_ptr(), c.data_ptr(), h,
                                           self._ef(coeff).ctypes.data, self._ef(yred).ctypes.data))
        return a

    def pcs_commit(self, field, hash_kind, evals_dev, log_blowup):
        """TwoAdicFriPcs::commit for one matrix over the subgroup H, fully device resident.
        Returns (lde tensor (h<<log_blowup, w) bit-reversed rows, digest layers)."""
        m = self._dev(evals_dev); self._use_torch_stream()
        h, w = int(m.shape[0]), int(m.shape[1])
        lde = self._empty((h << log_blowup, w))
        tot = self.merkle_total_digests(h << log_blowup)
        out = self._empty((tot, 8))
        lens = (C.c_size_t * 65)(); nl = C.c_size_t()
        check(self.L.p3gpu_pcs_commit_dev(self.h, field, hash_kind, m.data_ptr(), h, w, log_blowup, lde.data_ptr(), out.data_ptr(),
                                          lens, C.byref(nl)))
        layers, off = [], 0
        for k in range(nl.value):
            layers.append(out[off:off + lens[k]]); off += lens[k]
        return lde, layers


    # ------------------------------------------------------------------ Poseidon2 AIR (SURVEY 8f ranks 2-3)
    def p2air_set_constants(self, field, beginning_full, partial, ending_full):
        a = np.ascontiguousarray(beginning_full, dtype=np.uint32).ravel()
        b = np.ascontiguousarray(partial, dtype=np.uint32).ravel()
        c = np.ascontiguousarray(ending_full, dtype=np.uint32).ravel()
        assert a.size == 64 and c.size == 64
        check(self.L.p3gpu_p2air_set_constants(self.h, field, a.ctypes.data, b.ctypes.data, b.size, c.ctypes.data))
        self._air_cols = int(self.L.p3gpu_p2air_field_columns(field, b.size))

    def p2air_generate_trace(self, field, inputs_dev, vector_len=8):
        """(n_perms, 16) CUDA tensor -> vectorised trace (n_perms / vector_len, vector_len * columns)."""
        x = self._dev(inputs_dev); self._use_torch_stream()
        n = int(x.shape[0])
        out = self._empty((n // vector_len, vector_len * self._air_cols))
        check(self.L.p3gpu_p2air_generate_trace_dev(self.h, field, x.data_ptr(), n, out.data_ptr()))
        return out

    def p2air_generate_trace_cols(self, field, inputs_dev, col0, col1, vector_len=8):
        """Columns [col0, col1) of `p2air_generate_trace`'s output: (n_perms / vector_len, col1 - col0)."""
        x = self._dev(inputs_dev); self._use_torch_stream()
        n = int(x.shape[0])
        out = self._empty((n // vector_len, col1 - col0))
        check(self.L.p3gpu_p2air_generate_trace_cols_dev(self.h, field, vector_len, x.data_ptr(), n, col0, col1, out.data_ptr()))
        return out

    def p2air_quotient(self, field, lde_dev, log_trace_height, alpha, vector_len=8):
        """quotient values (H, 4) in natural order over GENERATOR * K, |K| = H = LDE height."""
        m = self._dev(lde_dev); self._use_torch_stream()
        H = int(m.shape[0]); log_h = H.bit_length() - 1
        assert int(m.shape[1]) == vector_len * self._air_cols
        q = self._empty((H, 4))
        check(self.L.p3gpu_p2air_quotient_dev(self.h, field, vector_len, m.data_ptr(), log_h, log_trace_height, self._ef(alpha).ctypes.data, q.data_ptr()))
        return q

    # ------------------------------------------------------------------ Keccak-f AIR
    @staticmethod
    def keccak_air_height(n_hashes: int) -> int:
        """(24 n).next_power_of_two(): the trace height of n permutations (1 for n = 0)."""
        return 1 << max(24 * int(n_hashes) - 1, 0).bit_length()

    def keccak_air_generate_trace(self, field, inputs_dev):
        """(n, 25) contiguous CUDA int64 tensor of u64 lanes (input[x + 5 y] = state[x][y]) -> the (H, 2633) trace, padding included."""
        import torch
        x = self._air_inputs(inputs_dev, torch.int64, 25); self._use_torch_stream()
        n = int(x.shape[0])
        out = self._empty((self.keccak_air_height(n), _lib.KECCAK_AIR_COLS))
        check(self.L.p3gpu_keccak_air_generate_trace_dev(self.h, field, x.data_ptr() if n else None, n, out.data_ptr()))
        return out

    def keccak_air_quotient(self, field, lde_dev, log_trace_height, alpha):
        """`_air_quotient_2n` of the Keccak AIR (2633 columns)."""
        return self._air_quotient_2n(self.L.p3gpu_keccak_air_quotient_dev, _lib.KECCAK_AIR_COLS, field, lde_dev, log_trace_height, alpha)

    # ------------------------------------------------------------------ Blake3 AIR
    def blake3_air_generate_trace(self, field, inputs_dev):
        """(n, 24) contiguous CUDA int32 tensor of u32 words (16 message words, 8 chaining-value words), n a power of two -> the
        (n, 9168) trace."""
        import torch
        x = self._air_inputs(inputs_dev, torch.int32, 24); self._use_torch_stream()
        n = int(x.shape[0])
        out = self._empty((n, _lib.BLAKE3_AIR_COLS))
        check(self.L.p3gpu_blake3_air_generate_trace_dev(self.h, field, x.data_ptr(), n, out.data_ptr()))
        return out

    def blake3_air_quotient(self, field, lde_dev, log_trace_height, alpha):
        """`_air_quotient_2n` of the Blake3 AIR (9168 columns)."""
        return self._air_quotient_2n(self.L.p3gpu_blake3_air_quotient_dev, _lib.BLAKE3_AIR_COLS, field, lde_dev, log_trace_height, alpha)

    def blake3_air_generate_trace_cols(self, field, inputs_dev, col0, col1):
        """Columns [col0, col1) of `blake3_air_generate_trace`'s output: (n, col1 - col0)."""
        import torch
        x = self._air_inputs(inputs_dev, torch.int32, 24)
        return self._air_trace_cols(lambda out: self.L.p3gpu_blake3_air_generate_trace_cols_dev(self.h, field, x.data_ptr(), int(x.shape[0]),
                                                                                               col0, col1, out), int(x.shape[0]), col0, col1)

    def blake3_air_quotient_sharded(self, field, group, col_starts, log_lde_height, log_trace_height, alpha):
        """`_air_quotient_sharded` of the Blake3 AIR."""
        return self._air_quotient_sharded(self.L.p3gpu_blake3_air_quotient_sharded_dev, field, group, col_starts, log_lde_height,
                                          log_trace_height, alpha)

    # ------------------------------------------------------------------ SHA-256 AIR
    def sha256_air_generate_trace(self, field, inputs_dev):
        """(n, 24) contiguous CUDA int32 tensor of u32 words (the 16-word block, the 8-word chaining state), n a power of two -> the
        (n, 7728) trace."""
        import torch
        x = self._air_inputs(inputs_dev, torch.int32, 24); self._use_torch_stream()
        n = int(x.shape[0])
        out = self._empty((n, _lib.SHA256_AIR_COLS))
        check(self.L.p3gpu_sha256_air_generate_trace_dev(self.h, field, x.data_ptr(), n, out.data_ptr()))
        return out

    def sha256_air_quotient(self, field, lde_dev, log_trace_height, alpha):
        """`_air_quotient_2n` of the SHA-256 AIR (7728 columns)."""
        return self._air_quotient_2n(self.L.p3gpu_sha256_air_quotient_dev, _lib.SHA256_AIR_COLS, field, lde_dev, log_trace_height, alpha)

    def sha256_air_generate_trace_cols(self, field, inputs_dev, col0, col1):
        """Columns [col0, col1) of `sha256_air_generate_trace`'s output: (n, col1 - col0)."""
        import torch
        x = self._air_inputs(inputs_dev, torch.int32, 24)
        return self._air_trace_cols(lambda out: self.L.p3gpu_sha256_air_generate_trace_cols_dev(self.h, field, x.data_ptr(), int(x.shape[0]),
                                                                                               col0, col1, out), int(x.shape[0]), col0, col1)

    def sha256_air_quotient_sharded(self, field, group, col_starts, log_lde_height, log_trace_height, alpha):
        """`_air_quotient_sharded` of the SHA-256 AIR."""
        return self._air_quotient_sharded(self.L.p3gpu_sha256_air_quotient_sharded_dev, field, group, col_starts, log_lde_height,
                                          log_trace_height, alpha)

    # ------------------------------------------------------------------ Poseidon1 AIR
    def p1air_set_constants(self, field, initial_full, terminal_full, mds_circ_col, first_round_constants, m_i, partial_rc,
                            sparse_first_row, v, rounds_p):
        """Poseidon1Air::new(full, partial) constants (Montgomery words) for this context; see p3gpu_p1air_set_constants."""
        a = [np.ascontiguousarray(x, dtype=np.uint32).ravel() for x in
             (initial_full, terminal_full, mds_circ_col, first_round_constants, m_i, partial_rc, sparse_first_row, v)]
        rp = int(rounds_p)
        sizes = (64, 64, 16, 16, 256, rp - 1, 16 * rp, 16 * rp)
        if any(x.size != s for x, s in zip(a, sizes)):
            raise _lib.P3GpuError(f"Poseidon1 constants of sizes {[x.size for x in a]}: need {list(sizes)}", _lib.EINVAL)
        check(self.L.p3gpu_p1air_set_constants(self.h, field, *[x.ctypes.data if x.size else None for x in a], rp))
        self._p1air_cols = int(self.L.p3gpu_p1air_columns(field, rp))

    def p1air_generate_trace(self, field, inputs_dev, vector_len=8):
        """(n_perms, 16) contiguous CUDA int32 tensor of Montgomery words, n_perms vector_len times a power of two -> the vectorised
        trace (n_perms / vector_len, vector_len * columns)."""
        import torch
        x = self._air_inputs(inputs_dev, torch.int32, 16); self._use_torch_stream()
        n = int(x.shape[0])
        rows = n // vector_len
        if n == 0 or n % vector_len or rows & (rows - 1):
            raise _lib.P3GpuError(f"{n} permutations: need {vector_len} times a power of two", _lib.EINVAL)
        out = self._empty((rows, vector_len * self._p1air_cols))
        check(self.L.p3gpu_p1air_generate_trace_dev(self.h, field, x.data_ptr(), n, out.data_ptr()))
        return out

    def p1air_quotient(self, field, lde_dev, log_trace_height, alpha, vector_len=8):
        """`_air_quotient_2n` of the Poseidon1 AIR (vector_len * columns)."""
        entry = lambda h, f, *rest: self.L.p3gpu_p1air_quotient_dev(h, f, vector_len, *rest)
        return self._air_quotient_2n(entry, vector_len * self._p1air_cols, field, lde_dev, log_trace_height, alpha)

    def p1air_generate_trace_cols(self, field, inputs_dev, col0, col1, vector_len=8):
        """Columns [col0, col1) of `p1air_generate_trace`'s output: (n_perms / vector_len, col1 - col0)."""
        import torch
        x = self._air_inputs(inputs_dev, torch.int32, 16)
        n = int(x.shape[0])
        return self._air_trace_cols(lambda out: self.L.p3gpu_p1air_generate_trace_cols_dev(self.h, field, vector_len, x.data_ptr(), n, col0, col1,
                                                                                          out), n // vector_len, col0, col1)

    def p1air_quotient_sharded(self, field, group, col_starts, log_lde_height, log_trace_height, alpha, vector_len=8):
        """`_air_quotient_sharded` of the Poseidon1 AIR with vector_len permutations per row."""
        entry = lambda h, f, *rest: self.L.p3gpu_p1air_quotient_sharded_dev(h, f, vector_len, *rest)
        return self._air_quotient_sharded(entry, field, group, col_starts, log_lde_height, log_trace_height, alpha)

    # ------------------------------------------------------------------ shared by the hand-written Keccak, Blake3 and Poseidon1 AIRs
    @staticmethod
    def _air_inputs(t, dtype, width):
        """A trace generator's inputs: a contiguous CUDA (n, width) tensor of `dtype`."""
        assert t.is_cuda and t.dtype == dtype and t.is_contiguous(), f"inputs: contiguous CUDA {str(dtype).removeprefix('torch.')} (n, {width})"
        assert t.dim() == 2 and int(t.shape[1]) == width
        return t

    def _air_trace_cols(self, launch, rows, col0, col1):
        """A trace generator's column window: a (rows, col1 - col0) device matrix filled by `launch(out pointer)`."""
        col0, col1 = int(col0), int(col1)
        if not 0 <= col0 <= col1:
            raise _lib.P3GpuError(f"column window [{col0}, {col1})", _lib.EINVAL)
        self._use_torch_stream()
        out = self._empty((rows, col1 - col0))
        check(launch(out.data_ptr() if col1 > col0 else None))
        return out

    def _air_quotient_sharded(self, entry, field, group, col_starts, log_lde_height, log_trace_height, alpha):
        """My row block's quotient values after the row-sharded commit: (R, 4), R = 2^log_lde_height / world, the bit-reversed slice
        `rank` (entry m is natural index bitrev(rank R + m)).  `group`: the _lib.PeerGroupStruct of the commit (its row block is
        read in place), `col_starts`: the commit's world + 1 column offsets; `entry`: the AIR's p3gpu_*_quotient_sharded_dev."""
        self._use_torch_stream()
        cs = (C.c_size_t * len(col_starts))(*[int(x) for x in col_starts])
        q = self._empty(((1 << log_lde_height) // int(group.world), 4))
        check(entry(self.h, field, C.byref(group), cs, log_lde_height, log_trace_height, self._ef(alpha).ctypes.data, q.data_ptr()))
        return q

    def _air_quotient_2n(self, entry, width, field, lde_dev, log_trace_height, alpha):
        """Quotient values (2^(log_trace_height + 1), 4) in natural order over GENERATOR * K from the first 2^(log_trace_height + 1)
        rows of the committed bit-reversed LDE of a `width`-column trace; `entry`: the AIR's p3gpu_*_air_quotient_dev."""
        m = self._dev(lde_dev); self._use_torch_stream()
        H = int(m.shape[0]); log_h = H.bit_length() - 1
        if H != 1 << log_h or int(m.shape[1]) != width:
            raise _lib.P3GpuError(f"LDE of shape {tuple(m.shape)}: need 2^k rows x {width}", _lib.EINVAL)
        q = self._empty((2 << log_trace_height, 4))
        check(entry(self.h, field, m.data_ptr(), log_h, log_trace_height, self._ef(alpha).ctypes.data, q.data_ptr()))
        return q

    # ------------------------------------------------------------------ any AIR as a constraint program
    def air_program_create(self, field, nodes, constraints, width, n_public):
        """Compile an expression DAG: nodes (n, 4) uint32 rows (op, a, b, imm), constraints: node indices in assertion order.
        Returns an AirProgramHandle (freed with the object)."""
        nd = np.ascontiguousarray(nodes, dtype=np.uint32).reshape(-1, 4)
        cs = np.ascontiguousarray(constraints, dtype=np.uint32).ravel()
        h = C.c_void_p()
        check(self.L.p3gpu_air_program_create(self.h, field, nd.ctypes.data, nd.shape[0], cs.ctypes.data, cs.size, width, n_public, C.byref(h)))
        return AirProgramHandle(self.L, h)

    def air_quotient(self, prog, lde_dev, log_quotient_size, log_trace_height, public_values, alpha):
        """Quotient values (2^log_quotient_size, 4) in natural order over GENERATOR * K from the first 2^log_quotient_size rows of the
        committed bit-reversed LDE.  public_values: Montgomery words."""
        m = self._dev(lde_dev); self._use_torch_stream()
        H = int(m.shape[0]); log_h = H.bit_length() - 1
        if H != 1 << log_h:
            raise _lib.P3GpuError(f"LDE height {H} is not a power of two", _lib.EINVAL)
        pv = np.ascontiguousarray(public_values, dtype=np.uint32).ravel()
        q = self._empty((1 << log_quotient_size, 4))
        check(self.L.p3gpu_air_quotient_dev(self.h, prog.h, m.data_ptr(), log_h, log_quotient_size, log_trace_height,
                                            pv.ctypes.data if pv.size else None, self._ef(alpha).ctypes.data, q.data_ptr()))
        return q

    def air_program_create_layout(self, field, nodes, constraints, layout):
        """air_program_create for a program that may read preprocessed and periodic columns: layout = (width, n_public,
        preprocessed_width, n_periodic)."""
        nd = np.ascontiguousarray(nodes, dtype=np.uint32).reshape(-1, 4)
        cs = np.ascontiguousarray(constraints, dtype=np.uint32).ravel()
        lay = np.ascontiguousarray(layout, dtype=np.uint32)
        assert lay.size == 4
        h = C.c_void_p()
        check(self.L.p3gpu_air_program_create_layout(self.h, field, nd.ctypes.data, nd.shape[0], cs.ctypes.data, cs.size, lay.ctypes.data,
                                                     C.byref(h)))
        return AirProgramHandle(self.L, h)

    def air_quotient_layout(self, prog, lde_dev, pre_lde_dev, periodic_dev, log_quotient_size, log_trace_height, public_values, alpha):
        """air_quotient with the preprocessed LDE (committed, bit-reversed; None without preprocessed columns) and the periodic table
        ((p_max * 2^q, n_periodic), natural order; None without periodic columns)."""
        m = self._dev(lde_dev); self._use_torch_stream()
        H = int(m.shape[0]); log_h = H.bit_length() - 1
        pre = self._dev(pre_lde_dev) if pre_lde_dev is not None else None
        per = self._dev(periodic_dev) if periodic_dev is not None else None
        for name, t in (("LDE", m), ("preprocessed LDE", pre), ("periodic table", per)):
            if t is not None and int(t.shape[0]) & (int(t.shape[0]) - 1):
                raise _lib.P3GpuError(f"{name} height {int(t.shape[0])} is not a power of two", _lib.EINVAL)
        pv = np.ascontiguousarray(public_values, dtype=np.uint32).ravel()
        q = self._empty((1 << log_quotient_size, 4))
        check(self.L.p3gpu_air_quotient_layout_dev(self.h, prog.h, m.data_ptr(), log_h,
                                                   pre.data_ptr() if pre is not None else None,
                                                   int(pre.shape[0]).bit_length() - 1 if pre is not None else 0,
                                                   per.data_ptr() if per is not None else None,
                                                   int(per.shape[0]).bit_length() - 1 if per is not None else 0,
                                                   log_quotient_size, log_trace_height, pv.ctypes.data if pv.size else None,
                                                   self._ef(alpha).ctypes.data, q.data_ptr()))
        return q

    def air_quotient_sharded(self, prog, group, col_starts, periodic_dev, log_lde_height, log_trace_height, public_values, alpha):
        """p3gpu_air_quotient_sharded_dev: my row block's quotient values after the row-sharded commit, over the LDE domain: (R, 4),
        R = 2^log_lde_height / world, the bit-reversed slice `rank`.  `group`: the _lib.PeerGroupStruct of the commit (every rank's row
        block: mine is read in place, the one holding my next rows too), `col_starts`: the commit's world + 1 column offsets,
        `periodic_dev`: the periodic table (None without periodic columns), public_values: Montgomery words."""
        self._use_torch_stream()
        per = self._dev(periodic_dev) if periodic_dev is not None else None
        if per is not None and int(per.shape[0]) & (int(per.shape[0]) - 1):
            raise _lib.P3GpuError(f"periodic table height {int(per.shape[0])} is not a power of two", _lib.EINVAL)
        cs = (C.c_size_t * len(col_starts))(*[int(x) for x in col_starts])
        pv = np.ascontiguousarray(public_values, dtype=np.uint32).ravel()
        q = self._empty(((1 << log_lde_height) // int(group.world), 4))
        check(self.L.p3gpu_air_quotient_sharded_dev(self.h, prog.h, C.byref(group), cs, per.data_ptr() if per is not None else None,
                                                    int(per.shape[0]).bit_length() - 1 if per is not None else 0, log_lde_height,
                                                    log_trace_height, pv.ctypes.data if pv.size else None, self._ef(alpha).ctypes.data,
                                                    q.data_ptr()))
        return q

    # ------------------------------------------------------------------ the debug constraint check (air.check_constraints)
    def air_check_program_create(self, field, nodes, constraints, layout):
        """A check program (p3gpu_air_check_program_create) of the DAG: layout = (width, n_public, preprocessed_width, n_periodic)."""
        nd = np.ascontiguousarray(nodes, dtype=np.uint32).reshape(-1, 4)
        cs = np.ascontiguousarray(constraints, dtype=np.uint32).ravel()
        lay = np.ascontiguousarray(layout, dtype=np.uint32)
        assert lay.size == 4
        h = C.c_void_p()
        check(self.L.p3gpu_air_check_program_create(self.h, field, nd.ctypes.data, nd.shape[0], cs.ctypes.data, cs.size, lay.ctypes.data,
                                                    C.byref(h)))
        return AirProgramHandle(self.L, h)

    def _check_args(self, trace_dev, pre_dev, periodic_dev, public_values):
        m = self._dev(trace_dev); self._use_torch_stream()
        pre = self._dev(pre_dev) if pre_dev is not None else None
        per = self._dev(periodic_dev) if periodic_dev is not None else None
        pv = np.ascontiguousarray(public_values, dtype=np.uint32).ravel()
        return (m.data_ptr(), int(m.shape[0]), pre.data_ptr() if pre is not None else None, per.data_ptr() if per is not None else None,
                int(per.shape[0]) if per is not None else 0), pv

    def air_check_counts(self, prog, trace_dev, pre_dev, periodic_dev, public_values):
        """Pass 1 of the check: (height,) int32, the number of constraints failing on each row of the (height, width) trace.
        pre_dev: the preprocessed trace (height rows); periodic_dev: the periodic columns repeated to the largest period; None when
        the AIR has none.  public_values: Montgomery words."""
        args, pv = self._check_args(trace_dev, pre_dev, periodic_dev, public_values)
        counts = self._empty((args[1],))
        check(self.L.p3gpu_air_check_dev(self.h, prog.h, *args, pv.ctypes.data if pv.size else None, counts.data_ptr()))
        return counts

    def air_check_rows(self, prog, trace_dev, pre_dev, periodic_dev, public_values, rows_dev, offsets_dev, n_failed):
        """Pass 2 of the check: (n_failed,) int32, the failing constraints of row rows_dev[j] (int32 CUDA) in ascending order from
        offsets_dev[j] (int64 CUDA) on."""
        import torch
        assert rows_dev.is_cuda and rows_dev.dtype == torch.int32 and rows_dev.is_contiguous()
        assert offsets_dev.is_cuda and offsets_dev.dtype == torch.int64 and offsets_dev.is_contiguous()
        assert int(offsets_dev.numel()) == int(rows_dev.numel())
        args, pv = self._check_args(trace_dev, pre_dev, periodic_dev, public_values)
        failed = self._empty((int(n_failed),))
        check(self.L.p3gpu_air_check_rows_dev(self.h, prog.h, *args, pv.ctypes.data if pv.size else None, rows_dev.data_ptr(),
                                              int(rows_dev.numel()), offsets_dev.data_ptr(), failed.data_ptr()))
        return failed

    def pcs_commit_host(self, field, hash_kind, evals_host, log_blowup, cap_height):
        """p3gpu_pcs_commit: TwoAdicFriPcs::commit with the trace in HOST memory (numpy uint32 array or pinned CPU int32 tensor);
        the LDE and the digest layers stay on the device, only the cap returns.  Returns (cap (n, 8) array, lde, layers)."""
        if _is_torch(evals_host):
            assert not evals_host.is_cuda and evals_host.is_contiguous()
            h, w, ptr = int(evals_host.shape[0]), int(evals_host.shape[1]), evals_host.data_ptr()
        else:
            m = self._np(evals_host)
            h, w, ptr = int(m.shape[0]), int(m.shape[1]), m.ctypes.data
        self._use_torch_stream()
        lde = self._empty((h << log_blowup, w))
        out = self._empty((self.merkle_total_digests(h << log_blowup), 8))
        lens = (C.c_size_t * 65)(); nl = C.c_size_t(); cap_len = C.c_size_t()
        cap = np.zeros((1 << cap_height, 8), dtype=np.uint32)
        check(self.L.p3gpu_pcs_commit(self.h, field, hash_kind, ptr, h, w, log_blowup, cap_height, lde.data_ptr(), out.data_ptr(), lens,
                                      C.byref(nl), cap.ctypes.data, C.byref(cap_len)))
        layers, off = [], 0
        for k in range(nl.value):
            layers.append(out[off:off + lens[k]]); off += lens[k]
        return cap[: cap_len.value].copy(), lde, layers


class AirProgramHandle:
    """A compiled constraint program (p3gpu_air_program); `info()` -> (instructions, slots, constraints)."""

    def __init__(self, L, h):
        self.L, self.h = L, h

    def info(self):
        n = [C.c_size_t() for _ in range(3)]
        check(self.L.p3gpu_air_program_info(self.h, *[C.byref(v) for v in n]))
        return tuple(int(v.value) for v in n)

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.L.p3gpu_air_program_destroy(self.h)
                self.h = None
        except Exception:
            pass


_default = {}


def default_gpu(device: int = 0) -> Gpu:
    if device not in _default:
        _default[device] = Gpu(device)
    return _default[device]
