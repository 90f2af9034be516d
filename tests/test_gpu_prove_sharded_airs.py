"""The row-sharded prove (distributed.prove_sharded) of the Blake3, SHA-256 and Poseidon1 AIRs over both fields, and of the Poseidon2
AIR under the Keccak configuration: on every rank the proof bytes equal the single-GPU `prove` on the whole trace, the verifier
accepts the proof and rejects a flipped byte.  Before the proof, each rank checks the pieces it is built from: `generate_trace_cols`
against column slices of the full trace (windows that cut a permutation, a 4-column unit, and the whole row), and its sharded
quotient slice against the matching rows of the dense kernel on the full LDE.

One process per rank with gloo bootstrap, as in test_gpu_prove_sharded.py (all ranks share cuda:0 on a one-GPU box), and world = 1
in this process.  The statements are tools/air_prove.py's (the example binary's inputs and constants) at 2^12 trace rows, with
new_benchmark_high_arity's FRI parameters.  Without peers, every AIR's sharded kernel also runs on the chunk-major row block a
world-4 commit leaves, built on one GPU (distributed.chunk_major_block): the layout a one-GPU machine otherwise never reads."""
import importlib.util
import os
import pathlib

import numpy as np
import pytest
import torch

from plonky3_b200 import _lib
from plonky3_b200.distributed import (PeerGroup, block_view, chunk_major_block, column_starts, prove_sharded,
                                      quotient_slice_natural_indices)
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.gpu import Gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import KeccakStarkConfig, StarkConfig, prove, verify

pytestmark = pytest.mark.gpu
ROOT = pathlib.Path(__file__).resolve().parent.parent
FIELDS = {"kb": KoalaBear, "bb": BabyBear}


def _air_prove():
    spec = importlib.util.spec_from_file_location("air_prove", ROOT / "tools" / "air_prove.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _statement(gpu, air_name, f, config_name, log_n, cap_height):
    """(config, air, device inputs) of tools/air_prove.py's statement at 2^log_n trace rows."""
    ap = _air_prove()
    make, _, hashes, random_inputs, dtype = ap.AIRS[air_name]
    if config_name == "keccak":
        m = MerkleTreeMmcs.keccak(f, cap_height=cap_height, gpu=gpu)
        config = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters.new_benchmark_high_arity(m)))
    else:
        p16, p24 = default_poseidon2(f, 16), default_poseidon2(f, 24)
        m = MerkleTreeMmcs.poseidon2(p16, p24, cap_height=cap_height, gpu=gpu)
        config = StarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters.new_benchmark_high_arity(m)), p24, 16)
    air = make(f, gpu)
    inputs = torch.from_numpy(np.ascontiguousarray(random_inputs(f, hashes(log_n))).view(dtype)).to(f"cuda:{gpu.device}")
    return config, air, inputs


def _windows(air, rank):
    """Windows that cut a 4-column unit, a permutation (Poseidon: 164 / 298 columns; hashes: a 32-bit word), and the whole row."""
    W = air.width()
    return [(0, 1), (2, 7), (100, 300), (161, 167), (295, 301), (5 + rank, W - 3), (0, W)]


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _check_pieces(air, inputs, full, rank, world, starts, bad):
    for a, b in [(starts[rank], starts[rank + 1])] + _windows(air, rank):
        if not torch.equal(air.generate_trace_cols(inputs, a, b), full[:, a:b]):
            bad.append(f"generate_trace_cols [{a}, {b}) differs from the column slice")


def _quotient_slice_check(air, full, log_n, q_mine, rank, world, bad, what):
    f, gpu = air.field, air.gpu
    alpha = np.array([f.to_monty(v) for v in (17 + log_n, 5, 7, 11)], dtype=np.uint32)
    lde = gpu.coset_lde_batch(f.id, full, 1, f.generator, bitrev_rows=True)
    q_full = _host(air.quotient_values(lde, log_n, alpha))
    got = _host(q_mine(alpha))
    nat = quotient_slice_natural_indices(rank, (2 << log_n) // world, log_n + 1)
    if not np.array_equal(got, q_full[nat]):
        rows = np.nonzero((got != q_full[nat]).any(axis=1))[0]
        bad.append(f"{what}: {rows.size} of {got.shape[0]} rows differ, first local row {rows[0]}")
    return lde


def _check_rank(gpu, rank, world, air_name, field, config_name, log_n, cap_height):
    """Everything one rank checks; returns a list of failure messages."""
    bad = []
    f = FIELDS[field]
    config, air, inputs = _statement(gpu, air_name, f, config_name, log_n, cap_height)
    full = air.generate_trace_rows(inputs)
    W, H = air.width(), 2 << log_n
    starts = column_starts(W, world, align=8)
    _check_pieces(air, inputs, full, rank, world, starts, bad)
    block = air.generate_trace_cols(inputs, starts[rank], starts[rank + 1])
    grp = PeerGroup(gpu, H // world, W, timeout_s=60.0)
    try:
        for p in config.pcs.mmcs.perms:
            p.upload(gpu)
        grp.commit(f, config.pcs.mmcs.hash_kind, block.contiguous(), starts, 1, cap_height)
        lde = _quotient_slice_check(air, full, log_n, lambda al: air.sharded_quotient_values(grp, log_n + 1, log_n, al), rank, world, bad,
                                    "sharded quotient")
        del lde
        expected = prove(config, air, full).to_postcard()
        proof = prove_sharded(config, air, grp, block, starts)
        raw = proof.to_postcard()
        if raw != expected:
            bad.append("prove_sharded bytes differ from prove")
        if rank == 0:
            verify(config, air, proof)
            flipped = bytearray(raw); flipped[len(raw) // 3] ^= 2
            try:
                verify(config, air, bytes(flipped))
                bad.append("a flipped byte was accepted")
            except Exception:                                    # noqa: BLE001 — any rejection
                pass
    finally:
        grp.close()
    return bad


def _rank_main(rank, world, port, case, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        import torch.distributed as dist
        device = rank if torch.cuda.device_count() >= world else 0
        torch.cuda.set_device(device)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        air_name, field, config_name, _, log_n, cap_height = case
        bad = _check_rank(Gpu(device), rank, world, air_name, field, config_name, log_n, cap_height)
        q.put((rank, not bad, "; ".join(bad)))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:                                       # noqa: BLE001 — surfaced by the parent
        import traceback
        q.put((rank, False, repr(e) + "\n" + traceback.format_exc()))


# (air, field, configuration, world, log_n, cap_height): every AIR, world 2 and 4, both configurations, cap_height 3 and 1 (with
# world 4: the cap below the sub-tree roots), the Poseidon2 AIR under the Keccak configuration
CASES = [
    ("blake3", "kb", "keccak", 2, 12, 3),
    ("sha256", "bb", "poseidon2", 2, 12, 3),
    ("poseidon1", "kb", "poseidon2", 4, 12, 1),
    ("poseidon1", "bb", "keccak", 4, 12, 3),
    ("sha256", "kb", "keccak", 4, 12, 1),
    ("poseidon2", "kb", "keccak", 2, 12, 3),
]


@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_prove_sharded_airs_equal_prove(case):
    import torch.multiprocessing as mp
    world = case[3]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + (os.getpid() % 200) + 11 * CASES.index(case)
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, case, q)) for r in range(world)]
    for p in procs: p.start()
    res = [q.get(timeout=900) for _ in range(world)]
    for p in procs: p.join(timeout=60)
    assert all(ok for _, ok, _ in res), "; ".join(f"rank {r}: {m}" for r, ok, m in sorted(res) if not ok)


@pytest.mark.parametrize("air_name,field,config_name", [("blake3", "bb", "poseidon2"), ("sha256", "kb", "keccak"),
                                                        ("poseidon1", "kb", "keccak"), ("poseidon1", "bb", "poseidon2")])
def test_prove_sharded_single_rank_equals_prove(air_name, field, config_name):
    """world == 1 in this process (no torch.distributed): the row block is the dense LDE, every exchange is a local copy."""
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    bad = _check_rank(Gpu(0), 0, 1, air_name, field, config_name, 12, 3)
    assert not bad, "; ".join(bad)


@pytest.mark.parametrize("air_name,field", [("blake3", "kb"), ("sha256", "bb"), ("poseidon1", "kb"), ("poseidon1", "bb")])
def test_sharded_quotient_on_a_world_4_block(air_name, field):
    """Every rank's chunk-major row block of a world-4 commit, laid out on one GPU: the sharded kernel reads it in place and
    writes the rank's slice of the dense kernel's quotient.  With 64-column chunks a BabyBear Poseidon1 permutation (298 columns)
    straddles chunk bounds."""
    gpu = Gpu(0)
    f = FIELDS[field]
    _, air, inputs = _statement(gpu, air_name, f, "keccak", 12, 3)
    full = air.generate_trace_rows(inputs)
    world, log_n = 4, 12
    R = (2 << log_n) // world
    starts = column_starts(air.width(), world, align=8)
    lde = gpu.coset_lde_batch(f.id, full, 1, f.generator, bitrev_rows=True)
    bad = []
    for rank in range(world):
        block = chunk_major_block(lde[rank * R:(rank + 1) * R], world, starts)
        view = type("BlockView", (), {"struct": block_view(world, rank, block), "col_starts": starts})()
        _quotient_slice_check(air, full, log_n, lambda al: air.sharded_quotient_values(view, log_n + 1, log_n, al), rank, world, bad,
                              f"rank {rank}")
    assert not bad, "; ".join(bad)
