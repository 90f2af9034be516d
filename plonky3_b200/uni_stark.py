"""uni-stark `prove` and `verify` with every data-parallel step on the GPU.  Mirrors uni-stark/src/prover.rs:87-442
(prove_with_preprocessed) and fri/src/prover.rs:43-160 (prove_fri) with the reference's names; host code is only the protocol
sequencing (the transcript's sponge itself runs on the device, challenger.py).  Non-ZK.

`prove` is the one protocol sequence, for any AIR in air.SymbolicAir's surface: public values, next-row openings, any number of
quotient chunks up to the blowup, preprocessed columns committed once by `setup_preprocessed`, periodic columns.  The AIR evaluates
its own quotient on the device: a plain SymbolicAir through the constraint-program kernel (p3gpu_air_quotient_dev /
p3gpu_air_quotient_layout_dev); poseidon2_air.VectorizedPoseidon2Air, the config-5 benchmark's AIR (`prove_prime_field_31 --field
koala-bear --objective poseidon-2-permutations --log-trace-length L -d radix-2-dit-parallel -m poseidon-2`),
keccak_air.KeccakAir, blake3_air.Blake3Air, sha256_air.Sha256Air and poseidon1_air.VectorizedPoseidon1Air through their
hand-written kernels.  With
`shard=distributed.ShardedTrace(...)` the same lines prove the Poseidon2 (KoalaBear), Blake3, SHA-256 and Poseidon1 AIRs and any
constraint-program AIR without preprocessed columns with the trace's columns split over several GPUs, the shard standing in for the
trace commit, the quotient values and the trace's row reads of the opening.

    trace (device)  --pcs.commit-->  trace cap ............................... p3gpu_coset_lde_batch_dev + p3gpu_merkle_commit_dev
    alpha <- transcript;  quotient values on GENERATOR * K ................... air.quotient_values (p3gpu_p2air_quotient_dev, ...)
    commit_quotient (2 chunks for degree 3) ................................... LDE + Merkle as above
    zeta <- transcript;  pcs.open: opened values + reduced openings .......... p3gpu_open_* / columnwise / rowwise dot kernels
    prove_fri: commit phase (fold + commit per round), grind, query openings . p3gpu_fri_fold_dev, p3gpu_challenger_grind,
                                                                               p3gpu_gather_rows_dev / p3gpu_merkle_paths_dev

RoundConstants, VectorizedPoseidon2Air and VECTOR_LEN live in poseidon2_air and are re-exported here, as are Poseidon1Constants and
VectorizedPoseidon1Air from poseidon1_air.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field as dc_field
from typing import List, Optional

import numpy as np

from .challenger import DuplexChallenger, SerializingChallenger32
from .dft import Radix2DitParallel, _log2_strict
from .fri import FriParameters, TwoAdicFriFolding, TwoAdicFriPcs, commit_phase
from .merkle_tree import MerkleTreeMmcs
from .poseidon2 import Poseidon2
from .poseidon2_air import VECTOR_LEN, RoundConstants, VectorizedPoseidon2Air  # noqa: F401  (re-exported)
from .poseidon1_air import Poseidon1Constants, VectorizedPoseidon1Air  # noqa: F401  (re-exported)


@dataclass
class StarkConfig:
    """uni-stark/src/config.rs:47-87: the PCS and the initial challenger state."""
    pcs: TwoAdicFriPcs
    challenger_perm: Poseidon2                    # DuplexChallenger<_, Perm24, 24, 16>
    challenger_rate: int = 16

    def initialise_challenger(self) -> DuplexChallenger:
        return DuplexChallenger(self.pcs.dft.field, self.challenger_perm, self.challenger_rate, self.pcs.dft.gpu)


@dataclass
class KeccakStarkConfig:
    """The Keccak configuration (examples/src/proofs.rs:82-124, types.rs:19-35): a Keccak MMCS (MerkleTreeMmcs.keccak) and the
    transcript SerializingChallenger32<F, HashChallenger<u8, Keccak256Hash, 32>>.  Its digests are [u64; 4], which the wire form
    writes as varints (proof_io.DIGEST_U64X4)."""
    pcs: TwoAdicFriPcs
    digest_codec: str = "u64x4"

    def initialise_challenger(self) -> SerializingChallenger32:
        return SerializingChallenger32.from_hasher([], self.pcs.dft.field, self.pcs.dft.gpu)


@dataclass
class Sha256StarkConfig:
    """The SHA-256 configurations (keccak-air/examples/prove_baby_bear_sha256.rs, prove_baby_bear_sha256_compress.rs): a SHA-256
    MMCS (MerkleTreeMmcs.sha256, either node compression) and the transcript SerializingChallenger32<F, HashChallenger<u8, Sha256,
    32>>.  Its digests are [u8; 32], which the wire form writes as 32 raw bytes (proof_io.DIGEST_U8X32)."""
    pcs: TwoAdicFriPcs
    digest_codec: str = "u8x32"

    def initialise_challenger(self) -> SerializingChallenger32:
        return SerializingChallenger32.from_hasher([], self.pcs.dft.field, self.pcs.dft.gpu, hasher="sha256")


@dataclass
class Proof:
    """uni-stark/src/proof.rs:19-62 + fri/src/proof.rs:12-24 as plain arrays (Montgomery words)."""
    trace_commit: np.ndarray
    quotient_commit: np.ndarray
    trace_local: np.ndarray                       # (width, 4)
    quotient_chunks: List[np.ndarray]             # per chunk (4, 4)
    commit_phase_commits: List[np.ndarray]
    commit_pow_witnesses: List[int]
    final_poly: np.ndarray
    query_pow_witness: int
    query_indices: List[int]
    input_openings: list                          # per round: (opened rows per matrix, paths)
    commit_phase_openings: list                   # per FRI round: (log_arity, sibling values (n, arity-1, 4), paths)
    degree_bits: int
    timings_ms: dict = dc_field(default_factory=dict)
    trace_next: Optional[np.ndarray] = None       # (width, 4) when the AIR reads the next row (uni-stark/src/proof.rs:52-56)
    preprocessed_local: Optional[np.ndarray] = None   # (preprocessed width, 4) when the AIR has preprocessed columns
    preprocessed_next: Optional[np.ndarray] = None    # ... and its preprocessed_next_row_columns() is not empty
    input_opening_indices: list = dc_field(default_factory=list)     # per input batch: the height-reduced query indices
    commit_phase_indices: list = dc_field(default_factory=list)      # per FRI round: the opened group index of every query
    digest_codec: str = "f8"                      # how the configuration's digests serialise (proof_io: "f8" [F; 8], "u64x4" [u64; 4], "u8x32" [u8; 32])

    def to_postcard(self) -> bytes:
        """The reference's wire form (`postcard::to_allocvec(&proof)`, uni-stark/tests/fib_air.rs:401-412)."""
        from .proof_io import proof_to_postcard
        return proof_to_postcard(self, digest=self.digest_codec)


@dataclass
class PreprocessedVerifierKey:
    """uni-stark/src/preprocessed.rs PreprocessedVerifierKey: what the verifier needs of the committed preprocessed trace."""
    width: int
    degree_bits: int
    commitment: np.ndarray


@dataclass
class PreprocessedProverData:
    """uni-stark/src/preprocessed.rs PreprocessedProverData: the preprocessed trace committed once (LDE and tree resident), reusable
    by every proof of the same AIR and height."""
    width: int
    degree_bits: int
    commitment: np.ndarray
    prover_data: object


def setup_preprocessed(config, air, degree_bits: int):
    """uni-stark/src/preprocessed.rs:46-91: commit the AIR's preprocessed trace on the trace domain of 2^degree_bits rows (same blowup
    as the trace).  Returns (PreprocessedProverData, PreprocessedVerifierKey), or None when the AIR has no preprocessed columns."""
    import torch
    width = air.preprocessed_width()
    if width == 0:
        return None
    trace = air.preprocessed_trace()
    if int(trace.shape[0]) != 1 << degree_bits:
        raise ValueError(f"preprocessed trace height {int(trace.shape[0])} must equal the trace degree 2^{degree_bits}")
    pcs = config.pcs
    gpu = pcs.dft.gpu
    if not isinstance(trace, torch.Tensor):
        trace = torch.from_numpy(np.ascontiguousarray(trace, dtype=np.uint32).view(np.int32))
        if isinstance(getattr(gpu, "device", None), int):
            trace = trace.to(f"cuda:{gpu.device}")
    commitment, data = pcs.commit([(pcs.natural_domain_for_degree(1 << degree_bits), trace)])
    return (PreprocessedProverData(width, degree_bits, commitment, data), PreprocessedVerifierKey(width, degree_bits, commitment))


def get_log_num_quotient_chunks(air) -> int:
    """uni-stark/src/symbolic.rs get_log_num_quotient_chunks: log2_ceil(max(constraint_degree, 2) - 1) (non-ZK)."""
    d = max(air.max_constraint_degree(), 2)
    return max(d - 2, 0).bit_length()


def verify(config, air, proof, public_values=(), *, preprocessed_vk: Optional[PreprocessedVerifierKey] = None):
    """uni-stark/src/verifier.rs:282-295 (verify_with_preprocessed).  Raises verifier.VerificationError."""
    from .verifier import verify as _verify
    if preprocessed_vk is None:
        return _verify(config, air, proof, public_values)
    return _verify(config, air, proof, public_values, preprocessed_vk=preprocessed_vk)


def prove(config, air, trace, public_values=(), *, shard=None, preprocessed: Optional[PreprocessedProverData] = None,
          check_constraints: bool = False) -> Proof:
    """uni-stark/src/prover.rs:87-442 (prove_with_preprocessed).  `config`: StarkConfig, KeccakStarkConfig or Sha256StarkConfig — every transcript
    call goes through the challenger it initialises.  `air`: an air.SymbolicAir, such as poseidon2_air.VectorizedPoseidon2Air,
    keccak_air.KeccakAir, blake3_air.Blake3Air, sha256_air.Sha256Air or poseidon1_air.VectorizedPoseidon1Air.  `trace`: device
    (CUDA int32) matrix of height 2^n.  `public_values`: canonical integers.

    `preprocessed`: setup_preprocessed's prover data, required iff the AIR has preprocessed columns; its commitment is observed
    after the trace's, and the preprocessed trace is opened last (at zeta, and zeta * omega unless preprocessed_next_row_columns() is
    empty).  Periodic columns need nothing here: the AIR evaluates them on the quotient domain.

    `shard`: a distributed.ShardedTrace when the trace's columns are split over ranks; `trace` is then this rank's column block,
    and every rank returns the proof of the whole trace.

    `check_constraints`: run air.check_constraints on the trace before committing it, as the reference's debug builds do
    (uni-stark/src/prover.rs:102-103), and raise air.ConstraintViolation naming the first failing row and its constraints.  Not
    with `shard` (the check reads whole rows)."""
    if check_constraints and shard is not None:
        raise ValueError("check_constraints needs whole trace rows: it does not take a column-sharded trace")
    import torch
    from . import extension as X
    pcs, f, gpu = config.pcs, config.pcs.dft.field, config.pcs.dft.gpu
    sync = torch.cuda.synchronize
    T = {}

    def span(name, t0):
        sync(); T[name] = (time.perf_counter() - t0) * 1e3

    public_values = [int(v) for v in public_values]
    if len(public_values) != air.num_public_values():
        raise ValueError(f"{len(public_values)} public values given, the AIR has {air.num_public_values()}")
    width = shard.width if shard is not None else int(trace.shape[1])
    if width != air.width():
        raise ValueError(f"trace width {width} differs from the AIR width {air.width()}")
    degree = int(trace.shape[0])
    log_degree = _log2_strict(degree)
    log_num_quotient_chunks = get_log_num_quotient_chunks(air)
    num_quotient_chunks = 1 << log_num_quotient_chunks
    pre_width = air.preprocessed_width()
    periodic = air.periodic_columns()
    if pre_width > 0 and preprocessed is None:
        raise ValueError(f"the AIR has {pre_width} preprocessed columns: call setup_preprocessed and pass its prover data")
    if preprocessed is not None:
        if preprocessed.width != pre_width:
            raise ValueError(f"preprocessed prover data of width {preprocessed.width}, the AIR has {pre_width} preprocessed columns")
        if preprocessed.degree_bits != log_degree:
            raise ValueError(f"preprocessed trace height 2^{preprocessed.degree_bits} differs from the trace height 2^{log_degree}")
    if periodic:
        from .air import periodic_column_error
        err = periodic_column_error(periodic, degree)
        if err:
            raise ValueError(err)
    if shard is not None and pre_width:
        raise ValueError("the row-sharded prove does not take preprocessed columns (it does take periodic columns)")
    if log_num_quotient_chunks > pcs.fri.log_blowup:
        # the quotient domain must lie inside the committed LDE (fast path of get_evaluations_on_domain); the reference asserts too
        raise ValueError(f"constraint degree {air.max_constraint_degree()} needs {num_quotient_chunks} quotient chunks: log_blowup "
                         f"{pcs.fri.log_blowup} < {log_num_quotient_chunks}")
    opens_next = len(air.main_next_row_columns()) > 0
    pre_next = pre_width > 0 and len(air.preprocessed_next_row_columns()) > 0
    if check_constraints:
        from .air import check_constraints as _check
        _check(air, trace, public_values)
    challenger = config.initialise_challenger()
    trace_domain = pcs.natural_domain_for_degree(degree)

    t0 = time.perf_counter()
    if shard is None:
        trace_commit, trace_data = pcs.commit([(trace_domain, trace)])                   # prover.rs:215
    else:
        trace_commit, trace_data = shard.commit(pcs, trace)
    span("commit to trace data", t0)

    challenger.observe_canonical(log_degree)                                             # log_ext_degree (non-ZK)       :224
    challenger.observe_canonical(log_degree)                                             # log_degree                    :225
    challenger.observe_canonical(pre_width)                                              # preprocessed_width            :226
    challenger.observe_cap(trace_commit)                                                 # :230
    if pre_width > 0:
        challenger.observe_cap(preprocessed.commitment)                                  # :231-232
    for v in public_values:                                                              # :236
        challenger.observe_canonical(v)
    alpha = challenger.sample_algebra_element()                                          # :258

    t0 = time.perf_counter()
    quotient_domain = (f.mul(trace_domain[0], f.generator), log_degree + log_num_quotient_chunks)      # create_disjoint_domain
    if shard is None:
        trace_on_quotient_domain = pcs.get_evaluations_on_domain(trace_data, 0, quotient_domain).bit_reverse_rows()
        pre_q = (pcs.get_evaluations_on_domain(preprocessed.prover_data, 0, quotient_domain).bit_reverse_rows()
                 if pre_width > 0 else None)                                               # :272
        quotient_flat = air.quotient_values(trace_on_quotient_domain, log_degree, alpha, public_values,   # natural order = flatten_to_base
                                            preprocessed_on_quotient_domain=pre_q)
    else:
        quotient_flat = shard.quotient_values(air, quotient_domain, alpha, public_values)
    span("compute quotient polynomial", t0)

    t0 = time.perf_counter()
    quotient_commit, quotient_data = pcs.commit_quotient(quotient_domain, quotient_flat, num_quotient_chunks)     # :319
    span("commit to quotient poly chunks", t0)
    challenger.observe_cap(quotient_commit)

    zeta = challenger.sample_algebra_element()                                           # :365
    t0 = time.perf_counter()
    trace_points = [zeta]
    zeta_next = None
    if opens_next or pre_next:                                                           # zeta * omega_N (trace_domain.next_point)
        zeta_next = X.ef_scale(f, np.asarray(zeta, dtype=np.uint32), f.two_adic_generator(log_degree))
    if opens_next:
        trace_points.append(zeta_next)
    rounds = [(trace_data, [trace_points]), (quotient_data, [[zeta]] * num_quotient_chunks)]
    input_mmcs = [shard or pcs.mmcs, pcs.mmcs]
    if pre_width > 0:                                                                    # the preprocessed round last (:379-391)
        rounds.append((preprocessed.prover_data, [[zeta, zeta_next] if pre_next else [zeta]]))
        input_mmcs.append(pcs.mmcs)
    opened_values, fri_inputs = pcs.open_values_and_fri_inputs(rounds, challenger, input_mmcs)
    span("open: evaluate + reduce", t0)

    t0 = time.perf_counter()
    fri = prove_fri(pcs, fri_inputs, challenger, rounds, input_mmcs)
    span("open: FRI", t0)

    return Proof(trace_commit=trace_commit, quotient_commit=quotient_commit, trace_local=opened_values[0][0][0],
                 quotient_chunks=[v[0] for v in opened_values[1]], commit_phase_commits=fri["commits"],
                 commit_pow_witnesses=fri["pow_witnesses"], final_poly=fri["final_poly"], query_pow_witness=fri["query_pow_witness"],
                 query_indices=fri["indices"], input_openings=fri["input_openings"], commit_phase_openings=fri["commit_phase_openings"],
                 degree_bits=log_degree, timings_ms=T, input_opening_indices=fri["input_opening_indices"],
                 commit_phase_indices=fri["commit_phase_indices"], trace_next=opened_values[0][0][1] if opens_next else None,
                 preprocessed_local=opened_values[2][0][0] if pre_width > 0 else None,
                 preprocessed_next=opened_values[2][0][1] if pre_next else None,
                 digest_codec=getattr(config, "digest_codec", "f8"))


def prove_fri(pcs: TwoAdicFriPcs, inputs: list, challenger: DuplexChallenger, prover_data_with_opening_points: list,
              input_mmcs: Optional[list] = None) -> dict:
    """fri/src/prover.rs:43-160.  `input_mmcs[k]` (default pcs.mmcs) opens input batch k: anything with get_max_height(data) and
    open_multi_batch(indices, data), such as the row-sharded trace distributed.ShardedTrace."""
    import torch
    params: FriParameters = pcs.fri
    f, gpu = pcs.dft.field, pcs.dft.gpu
    assert inputs and params.num_queries > 0
    log_global_max_height = _log2_strict(int(inputs[0].shape[0]))
    T = {}
    t0 = time.perf_counter()
    res = commit_phase(TwoAdicFriFolding(f, gpu), params, inputs, challenger, pcs.dft)
    torch.cuda.synchronize(); T["commit phase"] = (time.perf_counter() - t0) * 1e3
    for la in res.log_arities:
        challenger.observe_canonical(la)                                                 # :108-110
    t0 = time.perf_counter()
    pow_witness = challenger.grind(params.query_proof_of_work_bits)                      # :112
    T["grind"] = (time.perf_counter() - t0) * 1e3
    indices = [challenger.sample_bits(log_global_max_height) for _ in range(params.num_queries)]     # extra_query_index_bits = 0
    t0 = time.perf_counter()
    # open_inputs (:380-417): every committed batch at the (height-reduced) query indices
    input_openings, input_opening_indices, commit_phase_indices = [], [], []
    openers = input_mmcs or [pcs.mmcs] * len(prover_data_with_opening_points)
    for (data, _), mmcs in zip(prover_data_with_opening_points, openers):
        log_max_height = _log2_strict(mmcs.get_max_height(data))
        reduced = [i >> (log_global_max_height - log_max_height) for i in indices]
        input_openings.append(mmcs.open_multi_batch(reduced, data))
        input_opening_indices.append(reduced)
    # answer_queries (:308-378)
    commit_phase_openings, cur = [], list(indices)
    for la, data in zip(res.log_arities, res.data):
        group = [i >> la for i in cur]
        commit_phase_indices.append(group)
        rows, paths = params.mmcs.open_multi_batch(group, data)
        opened = rows[0].reshape(len(cur), 1 << la, 4)
        keep = np.array([[j for j in range(1 << la) if j != (i & ((1 << la) - 1))] for i in cur], dtype=np.int64)
        siblings = np.take_along_axis(opened, keep[:, :, None], axis=1)
        commit_phase_openings.append((la, siblings, paths))
        cur = group
    torch.cuda.synchronize(); T["query phase"] = (time.perf_counter() - t0) * 1e3
    return {"commits": res.commits, "pow_witnesses": res.pow_witnesses, "final_poly": res.final_poly, "query_pow_witness": pow_witness,
            "indices": indices, "input_openings": input_openings, "commit_phase_openings": commit_phase_openings, "log_arities": res.log_arities,
            "input_opening_indices": input_opening_indices, "commit_phase_indices": commit_phase_indices, "timings_ms": T}
