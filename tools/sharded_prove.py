"""Time distributed.prove_sharded against uni_stark.prove in the same run, and assert that both write the same proof bytes.

    python tools/sharded_prove.py [L] [reps]                             one GPU, world = 1 (the cost of the sharded machinery)
    torchrun --nproc_per_node G tools/sharded_prove.py [L] [reps]        one process per GPU, world = G
    python tools/sharded_prove.py 18 3 --air blake3 --field koala-bear --config keccak

--air poseidon2 (the default) is the config-5 statement: 2^L rows x 1312 KoalaBear columns, random round constants and inputs;
blake3, sha256 and poseidon1 are tools/air_prove.py's statements (the example binary's inputs).  --config poseidon2 (the default)
or keccak; new_benchmark_high_arity, cap_height 3.  Rank 0 prints one JSON line: card name, power limit, SM count, world, the
per-span times of `prove` (rank 0) and of `prove_sharded` (max over ranks), each the median over `reps` runs after one warm-up run.

    python tools/sharded_prove.py 18 --air sha256 --quotient-kernel-world 4 [--kernel-reps 10]

times, in one process on one GPU, the AIR's sharded quotient kernel on rank 0's chunk-major row block of a world-4 commit (R = 2^(L+1)
/ 4 rows, laid out by distributed.chunk_major_block and read in place) against the dense kernel on the same number of rows (the
trace of the first 2^L / 4 rows), CUDA events, median of --kernel-reps launches after a warm-up; checks the slice against the dense
kernel on the whole LDE first.  Blake3, SHA-256, Poseidon1 and the symbolic AIR.

    python tools/sharded_prove.py 18 3 --air symbolic [--degree 5 --log-blowup 2]

--air symbolic is a constraint-program SymbolicAir (tests/sharded_symbolic_examples.py wide_mul): 64 MulAir-style columns of
degree 3 at log_blowup 1 by default, whose transition constraints read the next row; --degree 5 --log-blowup 2 is its four-chunk
instance.  Its sharded quotient is p3gpu_air_quotient_sharded_dev, whose next rows come from one peer's row block (on one GPU that
"peer" is another block on the same device, so --quotient-kernel-world does not measure the link); the dense kernel is
p3gpu_air_quotient_dev."""
import argparse
import importlib.util
import json
import os
import pathlib
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]
import sharded_symbolic_examples as SYM
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.distributed import (PeerGroup, block_view, blocks_view, chunk_major_block, column_segments, column_starts, next_row_rank,
                                      prove_sharded, quotient_slice_natural_indices)
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import Gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import KeccakStarkConfig, RoundConstants, StarkConfig, VectorizedPoseidon2Air, prove

ap = argparse.ArgumentParser()
ap.add_argument("log_n", nargs="?", type=int, default=20)
ap.add_argument("reps", nargs="?", type=int, default=3)
ap.add_argument("--air", choices=["poseidon2", "blake3", "sha256", "poseidon1", "symbolic"], default="poseidon2")
ap.add_argument("--degree", type=int, default=3, help="--air symbolic: constraint degree (3 or 5)")
ap.add_argument("--log-blowup", type=int, default=1, help="--air symbolic: log_blowup (2 for --degree 5)")
ap.add_argument("--field", choices=["koala-bear", "baby-bear"], default="koala-bear")
ap.add_argument("--config", choices=["poseidon2", "keccak"], default="poseidon2")
ap.add_argument("--quotient-kernel-world", type=int, default=0, help="time the sharded quotient kernel on a block laid out for this world")
ap.add_argument("--kernel-reps", type=int, default=10)
a = ap.parse_args()
L, REPS = a.log_n, a.reps
LB = a.log_blowup if a.air == "symbolic" else 1
F = KoalaBear if a.field == "koala-bear" else BabyBear
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
device = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(device)
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("gloo")
gpu = Gpu(device)
if a.config == "keccak":
    mm = MerkleTreeMmcs.keccak(F, cap_height=3, gpu=gpu)
    cfg = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(F, gpu), mm, FriParameters(LB, 0, 3, 100, 0, 16, mm)))
else:
    mm = MerkleTreeMmcs.poseidon2(default_poseidon2(F, 16), default_poseidon2(F, 24), 3, gpu)
    cfg = StarkConfig(TwoAdicFriPcs(Radix2DitParallel(F, gpu), mm, FriParameters(LB, 0, 3, 100, 0, 16, mm)), default_poseidon2(F, 24), 16)


def _air_prove():
    spec = importlib.util.spec_from_file_location("air_prove", ROOT / "tools" / "air_prove.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def statement(log_n):
    """(air, device inputs) of a 2^log_n-row trace, the same on every rank."""
    if a.air == "poseidon2" and F is KoalaBear:
        rs = np.random.default_rng(7)
        air = VectorizedPoseidon2Air(F, RoundConstants(rs.integers(0, F.P, (4, 16), dtype=np.uint32), rs.integers(0, F.P, 20, dtype=np.uint32),
                                                       rs.integers(0, F.P, (4, 16), dtype=np.uint32)), gpu)
        g = torch.Generator(device=f"cuda:{device}"); g.manual_seed(11)
        return air, torch.randint(0, F.P, (8 << log_n, 16), device=f"cuda:{device}", dtype=torch.int32, generator=g)
    if a.air == "symbolic":              # the "inputs" are the trace itself
        trace = SYM.wide_mul_trace(F, 1 << log_n, degree=a.degree)
        return SYM.wide_mul(F, degree=a.degree, gpu=gpu), torch.from_numpy(trace.view(np.int32)).to(f"cuda:{device}")
    make, _, hashes, random_inputs, dtype = _air_prove().AIRS[a.air]
    x = np.ascontiguousarray(random_inputs(F, hashes(log_n))).view(dtype)
    return make(F, gpu), torch.from_numpy(x).to(f"cuda:{device}")


def card():
    q = subprocess.run(["nvidia-smi", f"--id={device}", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def median_spans(runs):
    return {k: float(np.median([r[k] for r in runs])) for k in runs[0]}


def events_median(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); e.synchronize()
        times.append(s.elapsed_time(e))
    return statistics.median(times)


def trace_rows(air, inputs):
    return inputs if a.air == "symbolic" else air.generate_trace_rows(inputs)


def trace_cols(air, inputs, c0, c1):
    return inputs[:, c0:c1].contiguous() if a.air == "symbolic" else air.generate_trace_cols(inputs, c0, c1)


def symbolic_quotient_kernel(G):
    """The sharded program kernel on rank 0's world-G block (every rank's block laid out on this GPU: the next rows come from the
    block of next_row_rank(0)) against p3gpu_air_quotient_dev on the same number of rows."""
    air, full = statement(L)
    alpha = np.array([F.to_monty(v) for v in (3, 5, 7, 11)], dtype=np.uint32)
    lde = gpu.coset_lde_batch(F.id, full, LB, F.generator, bitrev_rows=True)
    R = lde.shape[0] // G
    starts = column_starts(air.width(), G, align=8)
    blocks = [chunk_major_block(lde[g * R:(g + 1) * R], G, starts) for g in range(G)]
    q_full = air.quotient_values(lde, L, alpha).cpu().numpy()
    del lde
    torch.cuda.empty_cache()
    view = type("BlocksView", (), {"struct": blocks_view(G, 0, blocks), "col_starts": starts})()
    sharded = lambda: air.sharded_quotient_values(view, L + LB, L, alpha)
    assert np.array_equal(sharded().cpu().numpy(), q_full[quotient_slice_natural_indices(0, R, L + LB)]), "sharded slice differs"
    sharded_ms = events_median(sharded, a.kernel_reps)
    del blocks
    torch.cuda.empty_cache()
    log_small = L - (G.bit_length() - 1)
    small, small_full = statement(log_small)
    small_lde = gpu.coset_lde_batch(F.id, small_full, LB, F.generator, bitrev_rows=True)
    assert small_lde.shape[0] == R
    dense_ms = events_median(lambda: small.quotient_values(small_lde, log_small, alpha), a.kernel_reps)
    print(json.dumps({"card": card(), "air": a.air, "degree": a.degree, "log_blowup": LB, "field": a.field, "layout_world": G,
                      "block_rows": R, "width": air.width(), "next_rows_on_rank": next_row_rank(0, G, LB),
                      "segments": len(column_segments(G, starts, R)), "sharded_kernel_ms": round(sharded_ms, 3),
                      "dense_kernel_ms": round(dense_ms, 3), "sharded_over_dense": round(sharded_ms / dense_ms, 3), "slice_equal": True}))


def quotient_kernel(G):
    """The sharded kernel on rank 0's world-G block against the dense kernel on the same number of rows."""
    assert a.air != "poseidon2", "the kernel comparison covers the Blake3, SHA-256, Poseidon1 and symbolic AIRs"
    if a.air == "symbolic":
        return symbolic_quotient_kernel(G)
    air, inputs = statement(L)
    alpha = np.array([F.to_monty(v) for v in (3, 5, 7, 11)], dtype=np.uint32)
    full = air.generate_trace_rows(inputs)
    lde = gpu.coset_lde_batch(F.id, full, 1, F.generator, bitrev_rows=True)
    del full
    R = lde.shape[0] // G
    starts = column_starts(air.width(), G, align=8)
    block = chunk_major_block(lde[:R], G, starts)
    q_full = air.quotient_values(lde, L, alpha).cpu().numpy()
    del lde
    torch.cuda.empty_cache()
    view = type("BlockView", (), {"struct": block_view(G, 0, block), "col_starts": starts})()
    sharded = lambda: air.sharded_quotient_values(view, L + 1, L, alpha)
    assert np.array_equal(sharded().cpu().numpy(), q_full[quotient_slice_natural_indices(0, R, L + 1)]), "sharded slice differs"
    sharded_ms = events_median(sharded, a.kernel_reps)
    del block
    torch.cuda.empty_cache()
    log_small = L - (G.bit_length() - 1)
    small, small_inputs = statement(log_small)
    small_lde = gpu.coset_lde_batch(F.id, small.generate_trace_rows(small_inputs), 1, F.generator, bitrev_rows=True)
    assert small_lde.shape[0] == R
    dense_ms = events_median(lambda: small.quotient_values(small_lde, log_small, alpha), a.kernel_reps)
    print(json.dumps({"card": card(), "air": a.air, "field": a.field, "layout_world": G, "block_rows": R, "width": air.width(),
                      "segments": len(column_segments(G, starts, R)),
                      "sharded_kernel_ms": round(sharded_ms, 3), "dense_kernel_ms": round(dense_ms, 3),
                      "sharded_over_dense": round(sharded_ms / dense_ms, 3), "slice_equal": True}))


def prove_runs():
    air, inputs = statement(L)
    W = air.width()
    # single-GPU reference (every rank computes it; rank 0's times are reported)
    trace = trace_rows(air, inputs)
    ref_runs = []
    for i in range(REPS + 1):
        p = prove(cfg, air, trace)
        if i:
            ref_runs.append(dict(p.timings_ms, total=sum(p.timings_ms.values())))
    expected = p.to_postcard()
    del trace, p
    torch.cuda.empty_cache()

    starts = column_starts(W, world, align=8)
    block = trace_cols(air, inputs, starts[rank], starts[rank + 1])
    grp = PeerGroup(gpu, (1 << (L + LB)) // world, W, timeout_s=120.0)
    sh_runs = []
    for i in range(REPS + 1):
        p = prove_sharded(cfg, air, grp, block, starts)
        assert p.to_postcard() == expected, "prove_sharded wrote different proof bytes"
        if i:
            sh_runs.append(dict(p.timings_ms, total=sum(p.timings_ms.values())))
    grp.close()
    if rank == 0:
        print(json.dumps({"card": card(), "sm_count": torch.cuda.get_device_properties(device).multi_processor_count, "world": world,
                          "air": a.air, "field": a.field, "config": a.config, "log_n": L, "log_blowup": LB, "width": W, "reps": REPS,
                          "bytes_equal": True,
                          "prove_ms": median_spans(ref_runs), "prove_sharded_ms_max_over_ranks": median_spans(sh_runs)}))


if a.quotient_kernel_world:
    quotient_kernel(a.quotient_kernel_world)
else:
    prove_runs()
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
