"""The row-sharded multi-GPU prove (plonky3_b200.distributed.prove_sharded) of the config-5 Poseidon2 AIR: on every rank the proof
bytes equal the single-GPU `prove` on the whole trace (and, in the single-rank and the first two-rank case, the CPU replay), the
verifier accepts it and rejects a flipped byte.  Before the proof is compared, the pieces it is built from are checked on their own: the column-window trace
generation against column slices of the full trace, and every rank's sharded quotient slice against the matching rows of the
single-GPU quotient kernel on the full LDE.

One process per rank, as in test_gpu_sharded.py: gloo only bootstraps the CUDA IPC handles; all ranks share cuda:0 when the box
has one GPU.  The multi-rank cases start at 2^12 trace rows, the smallest height the sharded commit's column-block LDE takes
(p3gpu_commit_sharded_dev needs the tiled pipeline there), with one rank as with several.  The example binary's constants (SmallRng seed 1) and FRI parameters (new_benchmark_high_arity: 100 queries,
16 proof-of-work bits), cap_height 3, plus one world-4 case with cap_height 1 (cap below the sub-tree roots' level)."""
import os

import numpy as np
import pytest
import torch

from oracle import p3_oracle as O

from plonky3_b200 import _lib
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.distributed import PeerGroup, column_starts, prove_sharded, quotient_slice_natural_indices
from plonky3_b200.field import KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import Gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import Poseidon2
from plonky3_b200.uni_stark import RoundConstants, StarkConfig, VectorizedPoseidon2Air, prove, verify

pytestmark = pytest.mark.gpu
f = KoalaBear
NUM_QUERIES, POW_BITS = 100, 16


def _gpu_perm(pm):
    w = pm.width
    return Poseidon2.new(f, w, np.array(pm.rc_init)[: 4 * w].reshape(4, w), np.array(pm.rc_term)[: 4 * w].reshape(4, w),
                         np.array(pm.rc_int)[: pm.rounds_p], monty=True)


def _statement(gpu, log_n, cap_height):
    """(config, air, oracle pieces, permutation inputs on the device) of prove_prime_field_31's statement at 2^log_n rows."""
    rng = O.SmallRng(1)
    oair = O.air_from_rng(f.id, rng)
    o16 = O.perm_from_rng(f.id, 16, rng); o24 = O.perm_from_rng(f.id, 24, rng)
    p16, p24 = _gpu_perm(o16), _gpu_perm(o24)
    mmcs = MerkleTreeMmcs.poseidon2(p16, p24, cap_height=cap_height, gpu=gpu)
    pcs = TwoAdicFriPcs(Radix2DitParallel(f, gpu), mmcs, FriParameters(1, 0, 3, NUM_QUERIES, 0, POW_BITS, mmcs))
    config = StarkConfig(pcs, p24, 16)
    air = VectorizedPoseidon2Air(f, RoundConstants(np.array(oair.beg).reshape(4, 16), np.array(oair.part)[: oair.rounds_p],
                                                   np.array(oair.end).reshape(4, 16)), gpu)
    inputs = O.SmallRng(1).field(f.id, (8 << log_n) * 16).reshape(-1, 16)
    return config, air, (oair, o16, o24, inputs), torch.from_numpy(inputs.view(np.int32)).to(f"cuda:{gpu.device}")


def host(t):
    return t.cpu().numpy().view(np.uint32)


def _check_rank(gpu, rank, world, log_n, cap_height, replay=False):
    """Everything one rank checks; returns a list of failure messages."""
    bad = []
    config, air, (oair, o16, o24, inputs), inputs_dev = _statement(gpu, log_n, cap_height)
    full = air.generate_trace_rows(inputs_dev)
    W, N = air.width(), 1 << log_n
    H, log_h = 2 * N, log_n + 1
    starts = column_starts(W, world, align=8)
    c0, c1 = starts[rank], starts[rank + 1]
    block = air.generate_trace_cols(inputs_dev, c0, c1)
    if not torch.equal(block, full[:, c0:c1]):
        bad.append(f"generate_trace_cols [{c0}, {c1}) differs from the column slice")
    for a, b in [(0, 1), (100, 300), (163, 165), (5 + rank, W - 3), (0, W)]:    # windows cutting a permutation, the whole row
        if not torch.equal(air.generate_trace_cols(inputs_dev, a, b), full[:, a:b]):
            bad.append(f"generate_trace_cols [{a}, {b}) differs from the column slice")
    grp = PeerGroup(gpu, H // world, W, timeout_s=60.0)
    try:
        # the sharded quotient kernel on the committed row block, against the single-GPU kernel on the full LDE
        for p in config.pcs.mmcs.perms:
            p.upload(gpu)
        cap, _, _ = grp.commit(f, config.pcs.mmcs.hash_kind, block.contiguous(), starts, 1, cap_height)
        alpha = O.random_matrix(f.id, 1, 4, seed=17 + log_n)[0]
        lde = gpu.coset_lde_batch(f.id, full, 1, f.generator, bitrev_rows=True)
        q_full = host(gpu.p2air_quotient(f.id, lde, log_n, alpha))
        q_mine = host(grp.p2air_quotient(f, air.vector_len, log_h, log_n, alpha))
        nat = quotient_slice_natural_indices(rank, H // world, log_h)
        if not np.array_equal(q_mine, q_full[nat]):
            rows = np.nonzero((q_mine != q_full[nat]).any(axis=1))[0]
            bad.append(f"sharded quotient: {rows.size} of {H // world} rows differ, first local row {rows[0]}")
        del lde
        # the proof
        expected = prove(config, air, full).to_postcard()
        proof = prove_sharded(config, air, grp, block, starts)
        raw = proof.to_postcard()
        if raw != expected:
            bad.append("prove_sharded bytes differ from prove")
        if not np.array_equal(proof.trace_commit, cap):
            bad.append("trace commitment differs from PeerGroup.commit's cap")
        if set(proof.timings_ms) != {"commit to trace data", "compute quotient polynomial", "commit to quotient poly chunks",
                                     "open: evaluate + reduce", "open: FRI"}:
            bad.append(f"spans {sorted(proof.timings_ms)}")
        if rank == 0:
            from plonky3_b200.verifier import VerificationError
            verify(config, air, proof)
            flipped = bytearray(raw); flipped[len(raw) // 3] ^= 2
            try:
                verify(config, air, bytes(flipped))
                bad.append("a flipped byte was accepted")
            except VerificationError:
                pass
            if replay:
                import p2_prove_replay as R
                exp = R.prove(oair, o16, o24, inputs, num_queries=NUM_QUERIES, query_pow_bits=POW_BITS)
                if raw != R.to_wire_proof(exp).to_postcard():
                    bad.append("prove_sharded bytes differ from the CPU replay")
    finally:
        grp.close()
    return bad


def _rank_main(rank, world, port, log_n, cap_height, q):
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        import torch.distributed as dist
        device = rank if torch.cuda.device_count() >= world else 0
        torch.cuda.set_device(device)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        bad = _check_rank(Gpu(device), rank, world, log_n, cap_height, replay=(world, log_n) == (2, 12))
        q.put((rank, not bad, "; ".join(bad)))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:                                   # noqa: BLE001 — surfaced by the parent
        import traceback
        q.put((rank, False, repr(e) + "\n" + traceback.format_exc()))


@pytest.mark.parametrize("world,log_n,cap_height", [(2, 12, 3), (2, 13, 3), (4, 12, 3), (4, 12, 1)])
def test_prove_sharded_equals_prove(world, log_n, cap_height):
    import torch.multiprocessing as mp
    assert (2 << log_n) // world >= 1024
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29400 + (os.getpid() % 200) + 7 * world + log_n + cap_height
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, log_n, cap_height, q)) for r in range(world)]
    for p in procs: p.start()
    res = [q.get(timeout=900) for _ in range(world)]
    for p in procs: p.join(timeout=60)
    assert all(ok for _, ok, _ in res), "; ".join(f"rank {r}: {m}" for r, ok, m in sorted(res) if not ok)


def test_prove_sharded_single_rank_equals_prove():
    """world == 1 in this process (no torch.distributed): the row block is the dense LDE, every exchange is a local copy."""
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    bad = _check_rank(Gpu(0), 0, 1, 12, 3, replay=True)
    assert not bad, "; ".join(bad)
