"""The coset-blocked prove (coset_blocks.CosetBlockedTrace) against `uni_stark.prove` on one GPU.

For the Blake3, SHA-256 and Poseidon1 AIRs over both fields, the Poseidon2 AIR over KoalaBear and constraint-program AIRs that read the
next row, with public values and with periodic columns, under the Poseidon2, Keccak and SHA-256 configurations, at log_blowup 1 (two
cosets) and 2 (four): `prove(..., shard=CosetBlockedTrace(...)).to_postcard()` equals the resident-LDE proof byte for byte, at cap
heights inside and above the coset sub-trees, and `verify` accepts it.  On a trace of 2 GB the peak of torch's allocations stays within
twice the trace plus the stated allowance, below the trace plus its LDE."""
import importlib.util
import pathlib

import numpy as np
import pytest
import torch

import sharded_symbolic_examples as S
from plonky3_b200.coset_blocks import CosetBlockedTrace, coset_blocked_allowance_bytes, coset_blocked_memory_bytes, prove_coset_blocked
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import Gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig, prove, verify

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
FIELDS = {"kb": KoalaBear, "bb": BabyBear}


def _air_prove():
    spec = importlib.util.spec_from_file_location("air_prove", ROOT / "tools" / "air_prove.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _config(gpu, f, name, cap_height, log_blowup):
    if name == "keccak":
        m = MerkleTreeMmcs.keccak(f, cap_height=cap_height, gpu=gpu)
    elif name == "sha256":
        m = MerkleTreeMmcs.sha256(f, cap_height=cap_height, gpu=gpu)
    else:
        m = MerkleTreeMmcs.poseidon2(default_poseidon2(f, 16), default_poseidon2(f, 24), cap_height=cap_height, gpu=gpu)
    pcs = TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters(log_blowup, 0, 3, 100, 0, 16, m))
    if name == "keccak":
        return KeccakStarkConfig(pcs)
    if name == "sha256":
        return Sha256StarkConfig(pcs)
    return StarkConfig(pcs, default_poseidon2(f, 24), 16)


def _statement(gpu, air_name, f, log_n):
    """(air, device trace, public values, log_blowup) of a valid statement at 2^log_n rows."""
    if air_name in ("mul64-deg5", "fib32", "periodic"):
        if air_name == "mul64-deg5":
            air, trace, pubs, lb = S.wide_mul(f, degree=5, gpu=gpu), S.wide_mul_trace(f, 1 << log_n, degree=5), [], 2
        elif air_name == "fib32":
            (trace, pubs), air, lb = S.wide_fib_trace(f, 1 << log_n), S.wide_fib(f, gpu=gpu), 1
        else:
            air, trace, pubs, lb = S.periodic(f, gpu=gpu), S.periodic_trace(f, 1 << log_n), [], 1
        return air, torch.from_numpy(np.ascontiguousarray(trace).view(np.int32)).to(f"cuda:{gpu.device}"), pubs, lb
    make, _, hashes, random_inputs, dtype = _air_prove().AIRS[air_name]
    air = make(f, gpu)
    inputs = torch.from_numpy(np.ascontiguousarray(random_inputs(f, hashes(log_n))).view(dtype)).to(f"cuda:{gpu.device}")
    return air, air.generate_trace_rows(inputs), [], 1


CASES = [  # (air, field, config, log_n, cap_height); the sharded quotient kernels take blocks of at least 2^10 rows
    ("blake3", "kb", "keccak", 10, 3), ("blake3", "bb", "poseidon2", 10, 0),
    ("sha256", "kb", "sha256", 10, 1), ("sha256", "bb", "keccak", 11, 4),
    ("poseidon1", "kb", "poseidon2", 10, 3), ("poseidon1", "bb", "sha256", 10, 0),
    ("poseidon2", "kb", "keccak", 10, 2), ("poseidon2", "kb", "poseidon2", 11, 5),
    ("fib32", "kb", "poseidon2", 10, 3), ("fib32", "bb", "sha256", 11, 0),
    ("periodic", "bb", "keccak", 10, 1), ("periodic", "kb", "sha256", 12, 3),
    ("mul64-deg5", "kb", "keccak", 10, 0), ("mul64-deg5", "bb", "poseidon2", 11, 1), ("mul64-deg5", "kb", "sha256", 10, 4),
]


@pytest.mark.parametrize("air_name,field,config_name,log_n,cap_height", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_blocked_proof_equals_the_resident_lde_proof(air_name, field, config_name, log_n, cap_height):
    gpu, f = Gpu(0), FIELDS[field]
    air, trace, pubs, lb = _statement(gpu, air_name, f, log_n)
    config = _config(gpu, f, config_name, cap_height, lb)
    want = prove(config, air, trace.clone(), pubs).to_postcard()
    shard = CosetBlockedTrace(gpu, config, air)
    proof = prove(config, air, trace, pubs, shard=shard)
    assert proof.to_postcard() == want
    verify(config, air, proof, pubs)
    assert shard.blocks == 1 << lb


def test_peak_memory_is_twice_the_trace_plus_the_allowance():
    gpu, f, log_n = Gpu(0), KoalaBear, 16
    air, trace, pubs, lb = _statement(gpu, "sha256", f, log_n)
    trace_bytes = trace.numel() * 4
    assert trace_bytes >= 2 * 10**9
    config = _config(gpu, f, "keccak", 3, lb)
    want = prove(config, air, trace.clone(), pubs).to_postcard()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated() - trace_bytes            # everything but the trace
    torch.cuda.reset_peak_memory_stats()
    proof = prove_coset_blocked(config, air, trace, pubs)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert proof.to_postcard() == want
    plan = coset_blocked_memory_bytes(air, log_n, lb)
    assert plan == 2 * trace_bytes + coset_blocked_allowance_bytes(air.width(), log_n, lb)
    assert peak <= plan, (peak, plan)
    assert peak < trace_bytes * (1 + (1 << lb)), (peak, trace_bytes)
