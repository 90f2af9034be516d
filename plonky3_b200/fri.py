"""FRI prover-side surface on the GPU: FriParameters + compute_log_arity_for_round (fri/src/config.rs:10-207),
TwoAdicFriFolding.fold_matrix (fri/src/two_adic_pcs.rs:134-213), commit_phase (fri/src/prover.rs:192-286) and
TwoAdicFriPcs.commit (fri/src/two_adic_pcs.rs:300-363).  The Fiat-Shamir challenger stays on the host: per round only
the Merkle cap crosses PCIe (<= 2^cap_height x 32 bytes)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import List, Optional

import numpy as np

from .dft import Radix2DitParallel, _log2_strict, reverse_matrix_index_bits
from .field import Field
from .gpu import _is_torch
from .merkle_tree import MerkleTreeMmcs


@dataclass
class FriParameters:
    """fri/src/config.rs:10-23."""
    log_blowup: int
    log_final_poly_len: int
    max_log_arity: int
    num_queries: int
    commit_proof_of_work_bits: int
    query_proof_of_work_bits: int
    mmcs: MerkleTreeMmcs

    def blowup(self): return 1 << self.log_blowup
    def final_poly_len(self): return 1 << self.log_final_poly_len

    @classmethod
    def new_testing(cls, mmcs, log_final_poly_len):  # config.rs:76-86
        return cls(2, log_final_poly_len, 1, 2, 1, 1, mmcs)

    @classmethod
    def new_benchmark(cls, mmcs):  # config.rs:104-114
        return cls(1, 0, 1, 100, 0, 16, mmcs)

    @classmethod
    def new_benchmark_high_arity(cls, mmcs):  # config.rs:118-128
        return cls(1, 0, 3, 100, 0, 16, mmcs)


def compute_log_arity_for_round(log_current_height, next_input_log_height, log_final_height, max_log_arity):
    """fri/src/config.rs:180-207."""
    if max_log_arity <= 0:
        raise ValueError("max_log_arity must be at least 1 to guarantee folding progress")
    max_fold = log_current_height - log_final_height
    if next_input_log_height is not None:
        max_fold = min(max_fold, log_current_height - next_input_log_height)
    return min(max_fold, max_log_arity)


class TwoAdicFriFolding:
    """FriFoldingStrategy for the two-adic PCS (two_adic_pcs.rs:92-213)."""

    def __init__(self, field: Field, gpu):
        self.field, self.gpu = field, gpu

    def extra_query_index_bits(self): return 0

    def fold_matrix(self, beta, log_arity: int, m):
        """m: (rows, arity*4) base matrix = rows x arity EF4 values, bit-reversed order -> (rows, 4)."""
        return self.gpu.fri_fold(self.field.id, m, log_arity, beta)


@dataclass
class CommitPhaseResult:
    commits: list
    data: list
    log_arities: List[int]
    pow_witnesses: list
    final_poly: np.ndarray


def commit_phase(folding: TwoAdicFriFolding, params: FriParameters, inputs: list, challenger, dft: Radix2DitParallel) -> CommitPhaseResult:
    """fri/src/prover.rs:192-286.  inputs: EF4 vectors ((len,4) arrays/tensors) sorted by descending length, bit-reversed.
    challenger protocol: observe_cap(cap), grind(bits) -> witness, sample_algebra_element() -> 4 Montgomery words,
    observe_algebra_slice(vec)."""
    if params.max_log_arity <= 0:
        raise ValueError("max_log_arity must be at least 1 to guarantee folding progress")
    inputs = list(inputs)
    folded = inputs.pop(0)
    commits, data, log_arities, pow_witnesses = [], [], [], []
    log_final_height = params.log_blowup + params.log_final_poly_len
    field = folding.field
    while folded.shape[0] > params.blowup() * params.final_poly_len():
        log_cur = _log2_strict(int(folded.shape[0]))
        nxt = _log2_strict(int(inputs[0].shape[0])) if inputs else None
        log_arity = compute_log_arity_for_round(log_cur, nxt, log_final_height, params.max_log_arity)
        log_arities.append(log_arity)
        leaves = folded.reshape(folded.shape[0] >> log_arity, 4 << log_arity)      # RowMajorMatrix::new(folded, arity) + ExtensionMmcs
        commit, prover_data = params.mmcs.commit_matrix(leaves)
        challenger.observe_cap(commit)
        commits.append(commit)
        pow_witnesses.append(challenger.grind(params.commit_proof_of_work_bits))
        beta = np.asarray(challenger.sample_algebra_element(), dtype=np.uint32)
        folded = folding.fold_matrix(beta, log_arity, leaves)
        data.append(prover_data)
        if inputs and inputs[0].shape[0] == folded.shape[0]:
            # folded += beta^arity * input  (prover.rs:258-265)
            beta_pow = _ef_exp_power_of_2(field, beta, log_arity)
            folded = _ef_axpy(folding.gpu, field, folded, inputs.pop(0), beta_pow)
    fl = params.final_poly_len()
    final = folded[:fl]
    final = final.cpu().numpy().view(np.uint32) if _is_torch(final) else np.array(final, dtype=np.uint32)
    if fl > 1:
        final = dft.idft_algebra_batch(reverse_matrix_index_bits(final.reshape(fl, 4)).reshape(fl, 1, 4)).reshape(fl, 4)
    challenger.observe_algebra_slice(final)
    return CommitPhaseResult(commits, data, log_arities, pow_witnesses, final)


def _ef_mul_host(field: Field, a, b):
    """EF4 product of two single elements on the host (binomial_extension.rs:724-770); scalar transcript arithmetic only."""
    p = field.P
    x = [field.from_monty(int(v)) for v in a]; y = [field.from_monty(int(v)) for v in b]
    r = [0] * 7
    for i in range(4):
        for j in range(4):
            r[i + j] = (r[i + j] + x[i] * y[j]) % p
    out = [(r[i] + field.EXT_W * r[i + 4]) % p for i in range(3)] + [r[3]]
    return np.array([field.to_monty(v) for v in out], dtype=np.uint32)


def _ef_exp_power_of_2(field: Field, a, k: int):
    for _ in range(k):
        a = _ef_mul_host(field, a, a)
    return np.asarray(a, dtype=np.uint32)


def _ef_axpy(gpu, field: Field, acc, x, s):
    import torch
    to_dev = lambda t: t if _is_torch(t) else torch.from_numpy(np.ascontiguousarray(t, dtype=np.uint32).view(np.int32)).to(f"cuda:{gpu.device}")
    was_host = not _is_torch(acc)
    out = gpu.ef_axpy(field.id, to_dev(acc).contiguous(), to_dev(x).contiguous(), s)
    return out.cpu().numpy().view(np.uint32) if was_host else out


def split_evals(num_chunks: int, evals):
    """TwoAdicMultiplicativeCoset::split_evals (commit/src/domain.rs:257-290): chunk c takes rows c, c+num_chunks, ..."""
    _log2_strict(num_chunks)
    return [evals[c::num_chunks].contiguous() if _is_torch(evals) else np.ascontiguousarray(evals[c::num_chunks]) for c in range(num_chunks)]


def _row_steps(gpu, f: Field, mmcs, m):
    """The two steps of TwoAdicFriPcs.open_values_and_fri_inputs that read matrix `m`'s rows:
      low_coset_dot(h, weights, scale)                the opened values at one point: the weighted sum of the first h rows, scaled;
      reduce_rows(acc, alpha, terms, coeff_and_yred)  the reduced openings of `m` at each (1/(z - x), alpha offset, opened values)
                                                      of `terms`, added into the height's accumulator `acc`; coeff_and_yred(offset,
                                                      opened values) gives open_reduce's alpha^offset and Mred(z).
    An opener whose matrix rows are spread over ranks (distributed.ShardedTrace) supplies both; any other matrix is whole on this
    device."""
    if hasattr(mmcs, "reduce_rows"):
        return mmcs.low_coset_dot, mmcs.reduce_rows

    def low_coset_dot(h, weights, scale):
        return gpu.columnwise_dot(f.id, m[:h], weights, scale)

    def reduce_rows(acc, alpha, terms, coeff_and_yred):
        r = gpu.rowwise_dot(f.id, m, alpha)                                  # Mred(x) for every row
        for inv_denoms, offset, ys in terms:
            gpu.open_reduce(f.id, acc, r, inv_denoms, *coeff_and_yred(offset, ys))
    return low_coset_dot, reduce_rows


class TwoAdicFriPcs:
    """TwoAdicFriPcs<Val, Dft, InputMmcs, FriMmcs> — commit side (two_adic_pcs.rs:261-363)."""

    def __init__(self, dft: Radix2DitParallel, mmcs: MerkleTreeMmcs, fri: FriParameters):
        self.dft, self.mmcs, self.fri = dft, mmcs, fri

    def natural_domain_for_degree(self, degree: int):
        return (self.dft.field.ONE, _log2_strict(degree))      # (shift, log_size): TwoAdicMultiplicativeCoset

    def commit(self, evaluations: list):
        """evaluations: list of ((shift, log_size), matrix).  LDE onto GENERATOR*K, bit-reversed rows, MMCS commit."""
        f = self.dft.field
        ldes = []
        for (dshift, log_size), evals in evaluations:
            assert (1 << log_size) == evals.shape[0]
            shift = f.div(f.generator, dshift)                   # two_adic_pcs.rs:312
            ldes.append(self.dft.coset_lde_batch(evals, self.fri.log_blowup, shift).bit_reverse_rows())
        return self.mmcs.commit(ldes)

    def get_quotient_ldes(self, evaluations: list, num_chunks: int = 0):
        """two_adic_pcs.rs:326-345: the same LDE as commit, without committing."""
        f = self.dft.field
        return [self.dft.coset_lde_batch(ev, self.fri.log_blowup, f.div(f.generator, dshift)).bit_reverse_rows()
                for (dshift, log_size), ev in evaluations]

    def commit_quotient(self, quotient_domain, quotient_evaluations, num_chunks: int):
        """Pcs::commit_quotient default (commit/src/pcs/univariate.rs:98-119): split into num_chunks sub-cosets
        shift * h^i * K (domain.rs:243-255), LDE each, commit the batch."""
        f = self.dft.field
        shift, log_size = quotient_domain
        log_chunks = _log2_strict(num_chunks)
        h = f.two_adic_generator(log_size)
        subs = split_evals(num_chunks, quotient_evaluations)
        doms = [(f.mul(shift, f.pow(h, i)), log_size - log_chunks) for i in range(num_chunks)]
        return self.commit_ldes(self.get_quotient_ldes(list(zip(doms, subs)), num_chunks))

    def commit_ldes(self, ldes: list):
        min_height = 1 << self.fri.log_blowup
        for lde in ldes:
            if lde.shape[0] < min_height:
                raise ValueError(f"committed LDE height {lde.shape[0]} is smaller than the blowup factor {min_height}")
        return self.mmcs.commit(ldes)

    def open_values_and_fri_inputs(self, data_with_points: list, challenger, input_mmcs: Optional[list] = None):
        """The pre-FRI part of TwoAdicFriPcs::open (two_adic_pcs.rs:413-662) with the LDEs resident on the device.

        data_with_points: list of (prover_data, points_per_matrix) — prover_data a MerkleTree whose leaves are CUDA matrices
        (committed bit-reversed LDEs), points_per_matrix[i] the EF4 points (4 Montgomery words each) matrix i is opened at.
        `input_mmcs[k]` (default self.mmcs) holds round k's matrices, as in prove_fri; see `_row_steps` for an opener whose
        rows are spread over ranks.
        challenger protocol: observe_algebra_slice(ys), sample_algebra_element().
        Returns (all_opened_values[round][matrix][point] -> (width, 4) array, fri_inputs: list of (len, 4) CUDA vectors in
        descending length — the `fri_input` handed to prove_fri / commit_phase)."""
        from . import extension as X
        import torch
        f, gpu = self.dft.field, self.dft.gpu
        openers = input_mmcs or [self.mmcs] * len(data_with_points)
        rounds = [(mmcs.get_matrices(data), points, mmcs) for (data, points), mmcs in zip(data_with_points, openers)]
        for mats, points, _ in rounds:
            assert len(mats) == len(points), "each matrix should have a corresponding set of evaluation points"
        log_global_max_height = _log2_strict(max(int(m.shape[0]) for mats, _, _ in rounds for m in mats))
        # compute_inverse_denominators (:743-780): one vector per unique point, for the tallest matrix opened there
        max_lh = {}
        for mats, points, _ in rounds:
            for m, pts in zip(mats, points):
                for z in pts:
                    k = tuple(int(v) for v in z)
                    max_lh[k] = max(max_lh.get(k, 0), _log2_strict(int(m.shape[0])))
        inv_denoms, adjusted = {}, {}
        for k, lh in max_lh.items():
            z = np.array(k, dtype=np.uint32)
            inv_denoms[k], adjusted[k] = gpu.open_inv_denoms(f.id, lh, z, X.ef_inv(f, z))
        # opened values by barycentric interpolation of the low coset (:496-563; interpolation.rs:161-193).  The values stay on the
        # device for the transcript (observed there) and for Mred(z); one small copy brings them back for the proof.  The scale is
        # host arithmetic on the GPU's idle path after that copy, so it is computed once per (low coset size, point).
        all_opened, opened_dev, scales = [], [], {}
        for mats, points, mmcs in rounds:
            per_mat, per_mat_dev = [], []
            for m, pts in zip(mats, points):
                h = int(m.shape[0]) >> self.fri.log_blowup
                log_h = _log2_strict(h)
                low_coset_dot, _ = _row_steps(gpu, f, mmcs, m)
                per_pt, per_pt_dev = [], []
                for z in pts:
                    k = tuple(int(v) for v in z)
                    if (h, k) not in scales:
                        z = np.array(k, dtype=np.uint32)
                        g_pow_n = f.pow(f.generator, h)
                        denom_inv = f.inv(f.mul(g_pow_n, f.to_monty(h)))
                        scales[h, k] = X.ef_scale(f, X.ef_mul(f, z, X.ef_sub(f, X.ef_pow(f, z, 1 << log_h), X.ef_from_base(f, g_pow_n))), denom_inv)
                    ys_dev = low_coset_dot(h, adjusted[k], scales[h, k])
                    challenger.observe_algebra_slice(ys_dev)
                    per_pt_dev.append(ys_dev)
                    per_pt.append(ys_dev.cpu().numpy().view(np.uint32))
                per_mat.append(per_pt); per_mat_dev.append(per_pt_dev)
            all_opened.append(per_mat); opened_dev.append(per_mat_dev)
        alpha = np.asarray(challenger.sample_algebra_element(), dtype=np.uint32)

        def coeff_and_yred(offset, ys_dev):
            coeff = X.ef_pow(f, alpha, offset)                                   # alpha_pow_offset
            # Mred(z) = sum_i alpha^i y_i: the same row-wise dot kernel on the 4 coefficient rows of the opened values,
            # recombined with the basis (1, X, X^2, X^3) on the host
            yt = ys_dev.t().contiguous()                                         # (4, width)
            return coeff, X.ef_from_basis_rows(f, gpu.rowwise_dot(f.id, yt, alpha).cpu().numpy().view(np.uint32))
        # reduced openings per height (:598-660)
        num_reduced, reduced = {}, {}
        for (mats, points, mmcs), opened_round in zip(rounds, opened_dev):
            for m, pts, opened_mat in zip(mats, points, opened_round):
                H = int(m.shape[0]); lh = _log2_strict(H)
                if lh not in reduced:
                    reduced[lh] = torch.zeros((H, 4), dtype=torch.int32, device=m.device)
                    num_reduced[lh] = 0
                terms = []                                                       # (1/(z - x), alpha offset, opened values) per point
                for z, ys_dev in zip(pts, opened_mat):
                    terms.append((inv_denoms[tuple(int(v) for v in z)], num_reduced[lh], ys_dev))
                    num_reduced[lh] += int(m.shape[1])
                _, reduce_rows = _row_steps(gpu, f, mmcs, m)
                reduce_rows(reduced[lh], alpha, terms, coeff_and_yred)
        fri_inputs = [reduced[lh] for lh in sorted(reduced, reverse=True)]
        return all_opened, fri_inputs

    # ---- Pcs::open / Pcs::verify (two_adic_pcs.rs:413-715) as whole operations
    def open(self, data_with_points: list, challenger):
        """Pcs::open: opened values of every matrix at every point + the FRI opening proof (fri/src/proof.rs FriProof, as the dict
        proof_io / verifier use: multi-openings with pruned multiproofs).  `data_with_points` as in open_values_and_fri_inputs."""
        from .merkle_tree import prune_paths
        from .uni_stark import prove_fri
        opened, fri_inputs = self.open_values_and_fri_inputs(data_with_points, challenger)
        fri = prove_fri(self, fri_inputs, challenger, data_with_points)
        nq = len(fri["indices"])
        proof = {
            "commit_phase_commits": fri["commits"], "commit_pow_witnesses": fri["pow_witnesses"], "final_poly": fri["final_poly"],
            "query_pow_witness": fri["query_pow_witness"],
            "input_openings": [{"opened_values": [[rows[m][q] for m in range(len(rows))] for q in range(nq)], "proof": prune_paths(idx, paths)}
                               for (rows, paths), idx in zip(fri["input_openings"], fri["input_opening_indices"])],
            "commit_phase_openings": [{"log_arity": la, "sibling_values": [sib[q] for q in range(nq)], "proof": prune_paths(idx, paths)}
                                      for (la, sib, paths), idx in zip(fri["commit_phase_openings"], fri["commit_phase_indices"])],
        }
        return opened, proof

    def verify(self, commitments_with_opening_points: list, proof: dict, challenger):
        """Pcs::verify (two_adic_pcs.rs:684-715): `commitments_with_opening_points` = [(commitment, [((shift, log_size), [(z, values)])])]
        with z (4,) and values (width, 4) Montgomery words, in commitment order.  Raises verifier.VerificationError."""
        from .verifier import Ext, verify_fri
        e = Ext(self.dft.field)
        rounds = []
        for commit, mats in commitments_with_opening_points:
            rmats = []
            for (_, log_size), pts in mats:
                for _, ys in pts:
                    challenger.observe_algebra_slice(np.asarray(ys, dtype=np.uint32))
                rmats.append((log_size, [(e.ec(z), [e.ec(v) for v in np.asarray(ys, dtype=np.uint32).reshape(-1, 4)]) for z, ys in pts]))
            rounds.append((commit, rmats))
        verify_fri(e, self.fri, self.mmcs, proof, challenger, rounds)

    def get_evaluations_on_domain(self, prover_data, idx: int, domain):
        """two_adic_pcs.rs:376-403.  Fast path: the first |domain| rows of the committed bit-reversed LDE (domain shift =
        GENERATOR, |domain| <= LDE height).  Slow path (:390-403): un-bit-reverse, coset iDFT over GENERATOR*H' to recover the
        coefficients, truncate to the polynomial degree, zero-pad and coset DFT onto the requested domain."""
        from .dft import BitReversedMatrixView
        f = self.dft.field
        shift, log_size = domain
        size = 1 << log_size
        lde = self.mmcs.get_matrices(prover_data)[idx]
        if shift == f.generator and lde.shape[0] >= size:
            return BitReversedMatrixView(lde[:size])
        poly_height = int(lde.shape[0]) >> self.fri.log_blowup
        lde_mat = reverse_matrix_index_bits(lde)                              # natural order over GENERATOR * H'
        coeffs = self.dft.coset_idft_batch(lde_mat, f.generator)[:poly_height]
        width = int(coeffs.shape[1])
        if _is_torch(coeffs):
            import torch
            padded = torch.zeros((max(size, 0), width), dtype=coeffs.dtype, device=coeffs.device)
            n = min(size, poly_height)
            padded[:n] = coeffs[:n]
        else:
            padded = np.zeros((size, width), dtype=np.uint32)
            n = min(size, poly_height)
            padded[:n] = coeffs[:n]
        result = self.dft.coset_dft_batch(padded, shift)                      # natural order over shift * K
        return BitReversedMatrixView(reverse_matrix_index_bits(result))
