"""The row-sharded prove of constraint-program SymbolicAirs (p3gpu_air_quotient_sharded_dev, distributed.prove_sharded).

* Kernel level: every rank's chunk-major row block of a world-1/2/4/8 commit laid out on one GPU (distributed.chunk_major_block), with
  a view naming every rank's block (distributed.blocks_view), so next-row columns come from another rank's block where the owner
  arithmetic says so.  Each rank's slice, written over a poisoned buffer, must equal the dense kernel's rows word for word.
* Prove: world 2 and 4 as spawned processes with gloo (all ranks share cuda:0 on a one-GPU box) and world 1 in this process; on every
  rank the proof bytes equal `uni_stark.prove` on the whole trace, `verify` accepts the proof and rejects a flipped byte.
* Errors: every refusal of the entry point happens before any launch (the context's launch counter does not move)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import sharded_symbolic_examples as S
from plonky3_b200 import _lib
from plonky3_b200.air import ADD, MAIN_LOCAL, MUL, SymbolicAir
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.distributed import (PeerGroup, blocks_view, chunk_major_block, column_starts, next_row_rank, prove_sharded,
                                      quotient_slice_natural_indices)
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import Gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig, prove, verify

pytestmark = pytest.mark.gpu
FIELDS = {"kb": KoalaBear, "bb": BabyBear}
POISON = 0xFFFFFFFF                                    # not a canonical word of either field: every entry must be overwritten


def _air(name, f, gpu, log_n):
    """(air, host trace, public values, log_blowup) of a valid statement at 2^log_n rows."""
    if name == "mul64":
        return S.wide_mul(f, gpu=gpu), S.wide_mul_trace(f, 1 << log_n), [], 1
    if name == "mul64-deg5":
        return S.wide_mul(f, degree=5, gpu=gpu), S.wide_mul_trace(f, 1 << log_n, degree=5), [], 2
    if name == "fib32":
        trace, pubs = S.wide_fib_trace(f, 1 << log_n)
        return S.wide_fib(f, gpu=gpu), trace, pubs, 1
    return S.periodic(f, gpu=gpu), S.periodic_trace(f, 1 << log_n), [], 1


def _dev(gpu, host):
    return torch.from_numpy(np.ascontiguousarray(host).view(np.int32)).to(f"cuda:{gpu.device}")


def _host(t):
    return t.cpu().numpy().view(np.uint32)


def _alpha(f):
    return np.array([f.to_monty(v) for v in (19, 5, 7, 11)], dtype=np.uint32)


def _sharded(gpu, air, struct, starts, log_lde, log_n, pubs, alpha, out, periodic=None):
    """p3gpu_air_quotient_sharded_dev into `out`; returns its status."""
    gpu._use_torch_stream()
    cs = (C.c_size_t * len(starts))(*[int(x) for x in starts])
    pv = np.array([air.field.to_monty(int(v) % air.field.P) for v in pubs], dtype=np.uint32)
    return gpu.L.p3gpu_air_quotient_sharded_dev(gpu.h, air.program().h, C.byref(struct), cs, periodic.data_ptr() if periodic is not None else None,
                                                int(periodic.shape[0]).bit_length() - 1 if periodic is not None else 0, log_lde, log_n,
                                                pv.ctypes.data if pv.size else None, np.ascontiguousarray(alpha).ctypes.data, out.data_ptr())


# ---- kernel level ----------------------------------------------------------------------------------------------------------
KERNEL_CASES = [(air, fld, world) for air in ("mul64", "mul64-deg5", "fib32", "periodic") for fld in ("bb", "kb") for world in (1, 2, 4, 8)]


@pytest.mark.parametrize("air_name,field,world", KERNEL_CASES, ids=["-".join(map(str, c)) for c in KERNEL_CASES])
def test_every_rank_slice_equals_the_dense_kernel(air_name, field, world):
    gpu, f, log_n = Gpu(0), FIELDS[field], 12
    air, trace, pubs, lb = _air(air_name, f, gpu, log_n)
    log_lde = log_n + lb
    H, R = 1 << log_lde, (1 << log_lde) // world
    lde = gpu.coset_lde_batch(f.id, _dev(gpu, trace), lb, f.generator, bitrev_rows=True)
    alpha = _alpha(f)
    dense = _host(air.quotient_values(lde, log_n, alpha, pubs))
    starts = column_starts(air.width(), world, align=8)
    blocks = [chunk_major_block(lde[g * R:(g + 1) * R], world, starts) for g in range(world)]
    periodic = air.periodic_table(log_n, log_lde)
    bad = []
    for g in range(world):
        out = torch.full((R, 4), -1, dtype=torch.int32, device="cuda:0")
        rc = _sharded(gpu, air, blocks_view(world, g, blocks), starts, log_lde, log_n, pubs, alpha, out, periodic)
        assert rc == 0, _lib.load().p3gpu_last_error()
        got = _host(out)
        assert not (got == POISON).any(), f"rank {g}: {int((got == POISON).sum())} words not written"
        exp = dense[quotient_slice_natural_indices(g, R, log_lde)]
        if not np.array_equal(got, exp):
            rows = np.nonzero((got != exp).any(axis=1))[0]
            bad.append(f"rank {g} (next rows on rank {next_row_rank(g, world, lb)}): {rows.size} of {R} rows differ, first {rows[0]}")
    assert H == lde.shape[0] and not bad, "; ".join(bad)


def test_the_python_surface_matches_the_entry_point():
    """SymbolicAir.sharded_quotient_values on a world-4 view: the same slice, public values passed through."""
    gpu, f, log_n = Gpu(0), BabyBear, 12
    air, trace, pubs, _ = _air("fib32", f, gpu, log_n)
    lde = gpu.coset_lde_batch(f.id, _dev(gpu, trace), 1, f.generator, bitrev_rows=True)
    dense = _host(air.quotient_values(lde, log_n, _alpha(f), pubs))
    world, R = 4, (2 << log_n) // 4
    starts = column_starts(air.width(), world, align=8)
    blocks = [chunk_major_block(lde[g * R:(g + 1) * R], world, starts) for g in range(world)]
    for g in range(world):
        view = type("View", (), {"struct": blocks_view(world, g, blocks), "col_starts": starts})()
        got = _host(air.sharded_quotient_values(view, log_n + 1, log_n, _alpha(f), pubs))
        assert np.array_equal(got, dense[quotient_slice_natural_indices(g, R, log_n + 1)])


# ---- prove -------------------------------------------------------------------------------------------------------------------
def _config(gpu, f, name, cap_height, log_blowup):
    if name == "keccak":
        m = MerkleTreeMmcs.keccak(f, cap_height=cap_height, gpu=gpu)
    elif name == "sha256":
        m = MerkleTreeMmcs.sha256(f, cap_height=cap_height, gpu=gpu)
    else:
        m = MerkleTreeMmcs.poseidon2(default_poseidon2(f, 16), default_poseidon2(f, 24), cap_height=cap_height, gpu=gpu)
    fri = FriParameters(log_blowup, 0, 3, 100, 0, 16, m)
    pcs = TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, fri)
    if name == "keccak":
        return KeccakStarkConfig(pcs)
    if name == "sha256":
        return Sha256StarkConfig(pcs)
    return StarkConfig(pcs, default_poseidon2(f, 24), 16)


def _check_rank(gpu, rank, world, air_name, field, config_name, log_n, cap_height):
    bad = []
    f = FIELDS[field]
    air, trace, pubs, lb = _air(air_name, f, gpu, log_n)
    config = _config(gpu, f, config_name, cap_height, lb)
    full = _dev(gpu, trace)
    W, H = air.width(), 1 << (log_n + lb)
    starts = column_starts(W, world, align=8)
    block = full[:, starts[rank]:starts[rank + 1]].contiguous()
    grp = PeerGroup(gpu, H // world, W, timeout_s=60.0)
    try:
        for p in config.pcs.mmcs.perms:
            p.upload(gpu)
        expected = prove(config, air, full, pubs).to_postcard()
        proof = prove_sharded(config, air, grp, block, starts, pubs)
        raw = proof.to_postcard()
        if raw != expected:
            bad.append("prove_sharded bytes differ from prove")
        if rank == 0:
            verify(config, air, proof, pubs)
            flipped = bytearray(raw); flipped[len(raw) // 3] ^= 2
            try:
                verify(config, air, bytes(flipped), pubs)
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


# (air, field, configuration, world, log_n, cap_height): next-row reads from a peer (world 4 at log_blowup 1), public values,
# periodic columns, all three configurations, the cap below the sub-tree roots (cap_height 1 < log2 4)
CASES = [
    ("mul64", "kb", "poseidon2", 2, 12, 3),
    ("fib32", "bb", "keccak", 4, 12, 1),
    ("periodic", "kb", "sha256", 4, 12, 3),
    ("mul64-deg5", "bb", "keccak", 4, 12, 1),
]


@pytest.mark.parametrize("case", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_prove_sharded_symbolic_equals_prove(case):
    import torch.multiprocessing as mp
    world = case[3]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29800 + (os.getpid() % 150) + 13 * CASES.index(case)
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, case, q)) for r in range(world)]
    for p in procs: p.start()
    res = [q.get(timeout=900) for _ in range(world)]
    for p in procs: p.join(timeout=60)
    assert all(ok for _, ok, _ in res), "; ".join(f"rank {r}: {m}" for r, ok, m in sorted(res) if not ok)


@pytest.mark.parametrize("air_name,field,config_name", [("periodic", "bb", "poseidon2"), ("fib32", "kb", "sha256"),
                                                        ("mul64-deg5", "kb", "poseidon2")])
def test_prove_sharded_symbolic_single_rank(air_name, field, config_name):
    """world == 1 in this process: the row block is the dense LDE, every exchange a local copy."""
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    bad = _check_rank(Gpu(0), 0, 1, air_name, field, config_name, 12, 3)
    assert not bad, "; ".join(bad)


# ---- errors before any launch ----------------------------------------------------------------------------------------------
def _many_slots_air(f, width, live):
    """`live` products kept alive until the last constraint (their sum), padded to 2048 constraints: about `live` slots."""
    def ev(b):
        m = b.main()
        ys = [m.local[k] * m.local[k] for k in range(live)]
        for y in ys:
            b.assert_zero(y)
        acc = ys[0]
        for y in ys[1:]:
            acc = acc + y
        b.assert_zero(acc)
        for _ in range(2048 - live - 1):
            b.assert_zero(m.local[0])
    return ev


def test_errors_are_refused_before_any_launch():
    gpu, f, log_n = Gpu(0), KoalaBear, 12
    air, trace, pubs, _ = _air("fib32", f, gpu, log_n)
    log_lde, world = log_n + 1, 4
    R = (1 << log_lde) // world
    starts = column_starts(32, world, align=8)
    blocks = [torch.zeros(R * 32 + 1, dtype=torch.int32, device="cuda:0") for _ in range(world)]
    view = blocks_view(world, 1, blocks)
    out = torch.zeros((R + 1, 4), dtype=torch.int32, device="cuda:0")
    alpha = _alpha(f)
    air.program()
    gpu.sync()

    def refused(code, match, **kw):
        args = dict(air=air, struct=view, starts=starts, log_lde=log_lde, log_n=log_n, pubs=pubs, alpha=alpha, out=out)
        args.update(kw)
        before = gpu.launches
        rc = _sharded(gpu, args["air"], args["struct"], args["starts"], args["log_lde"], args["log_n"], args["pubs"], args["alpha"],
                      args["out"])
        msg = _lib.load().p3gpu_last_error().decode()
        assert rc == code, (rc, msg)
        assert match in msg, msg
        assert gpu.launches == before, "launched before refusing"

    check_air = S.wide_fib(f, gpu=gpu)
    check_air._program = check_air.check_program()                  # a program created for the check
    refused(_lib.EINVAL, "p3gpu_air_check_program_create", air=check_air)
    refused(_lib.EINVAL, "alpha is not a canonical", alpha=np.array([f.P, 0, 0, 0], dtype=np.uint32))
    bad_pub = SymbolicAir(f, 32, S.wide_fib_eval(), num_public_values=3, max_constraint_degree=3, gpu=gpu)
    before = gpu.launches
    cs = (C.c_size_t * len(starts))(*starts)
    pv = np.array([0, f.P, 0], dtype=np.uint32)
    rc = gpu.L.p3gpu_air_quotient_sharded_dev(gpu.h, bad_pub.program().h, C.byref(view), cs, None, 0, log_lde, log_n, pv.ctypes.data,
                                              alpha.ctypes.data, out.data_ptr())
    assert rc == _lib.EINVAL and "public value 1 is not a canonical" in _lib.load().p3gpu_last_error().decode()
    assert gpu.launches == before
    refused(_lib.EINVAL, "misaligned quotient slice", out=out.view(-1)[1:])
    skewed = blocks_view(world, 1, blocks)
    skewed.rows[2] = blocks[2].data_ptr() + 2
    refused(_lib.EINVAL, "misaligned row block of rank 2", struct=skewed)
    refused(_lib.EINVAL, "does not start and end on a multiple of 8 columns", starts=[0, 4, 8, 16, 32])
    refused(_lib.EINVAL, "the column blocks cover 24 columns, the trace has 32", starts=[0, 8, 16, 24, 24])
    refused(_lib.EUNSUPPORTED, "at least 1024 rows per rank", log_lde=11, log_n=10)
    refused(_lib.EUNSUPPORTED, "the quotient domain is the LDE domain", log_lde=13, log_n=4)
    wide = SymbolicAir(f, 8000, _many_slots_air(f, 8000, 380), gpu=gpu)
    _, slots, cons = (int(x) for x in _info(gpu, wide.program()))
    assert cons == 2048 and cons * 16 + slots * 512 <= 227 * 1024 < cons * 16 + slots * 512 + 1000 * 8
    refused(_lib.EUNSUPPORTED, f"{slots} slots x 512 B + 2048 constraints x 16 B + 1000 units x 8 B", air=wide, starts=[0, 8000],
            struct=blocks_view(1, 0, blocks[:1]), pubs=[])


def _info(gpu, prog):
    n = [C.c_size_t() for _ in range(3)]
    assert gpu.L.p3gpu_air_program_info(prog.h, *[C.byref(x) for x in n]) == 0
    return [x.value for x in n]
