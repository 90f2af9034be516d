"""Times the constraint-program quotient kernel (p3gpu_air_quotient_dev) on an H100.

    poseidon2   the DSL's vectorised Poseidon2 AIR against the hand-written p3gpu_p2air_quotient_dev at the config-5 shape (trace
                2^log_n x 1312, blowup 2: LDE 2^(log_n + 1) x 1312), asserting equal output
    mul_air     MulAir (degree 3, boundary and transition constraints, 60 columns) at 2^log_n rows, blowup 4, quotient over 2^(log_n + 1)
                rows: ms and trace-read GB/s (local + next rows, each LDE word read once per row it belongs to)
    mul_air_pre MulAir with its coefficients in 20 preprocessed columns (a^2 b k - c, boundary a^2 + 1 = b) and its transition step
                in two periodic columns (a' = a + u + v, periods 4 and 16), same shape: ms and GB/s of trace reads (main local + next
                rows, preprocessed local rows; the periodic table is cache-resident and not counted)

Prints one JSON line per measurement.  CUDA-event timing, median of --reps after --warmup launches.

    python tools/air_program_bench.py [--log-n 20] [--reps 10] [--warmup 3] [--only poseidon2,mul_air,mul_air_pre]
"""
import argparse
import json
import pathlib
import sys

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import air_examples as E                                     # noqa: E402
from plonky3_b200.air import SymbolicAir                     # noqa: E402
from plonky3_b200.field import KoalaBear                     # noqa: E402
from plonky3_b200.gpu import default_gpu                     # noqa: E402
from plonky3_b200.poseidon2_air import RoundConstants, VectorizedPoseidon2Air, poseidon2_eval      # noqa: E402


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="poseidon2,mul_air,mul_air_pre")
    args = ap.parse_args()
    only = set(args.only.split(","))
    f, gpu = KoalaBear, default_gpu(0)
    name = torch.cuda.get_device_name(0)
    rng = np.random.default_rng(1)
    alpha = f.to_monty_array(rng.integers(0, f.P, 4).astype(np.uint64)).astype(np.uint32)

    if "poseidon2" in only:
        poseidon2(args, f, gpu, name, rng, alpha)
    if "mul_air" in only:
        mul_air(args, f, gpu, name, rng, alpha)
    if "mul_air_pre" in only:
        mul_air_pre(args, f, gpu, name, rng, alpha)


def poseidon2(args, f, gpu, name, rng, alpha):
    # Poseidon2: DSL program vs the hand-written kernel
    rcs = RoundConstants(f.to_monty_array(rng.integers(0, f.P, (4, 16)).astype(np.uint64)),
                         f.to_monty_array(rng.integers(0, f.P, 20).astype(np.uint64)), f.to_monty_array(rng.integers(0, f.P, (4, 16)).astype(np.uint64)))
    hand = VectorizedPoseidon2Air(f, rcs, gpu)
    ev, width = poseidon2_eval(f, rcs)
    dsl = SymbolicAir(f, width, ev, main_next_row_columns=[], gpu=gpu)
    inputs = torch.from_numpy(rng.integers(0, f.P, (8 << args.log_n, 16), dtype=np.uint32).view(np.int32)).cuda()
    trace = hand.generate_trace_rows(inputs)
    del inputs
    lde = gpu.coset_lde_batch(f.id, trace, 1, f.generator)
    del trace
    q_hand = hand.quotient_values(lde, args.log_n, alpha)
    q_dsl = dsl.quotient_values(lde, args.log_n, alpha)
    assert torch.equal(q_hand, q_dsl), "DSL Poseidon2 quotient differs from p3gpu_p2air_quotient_dev"
    del q_hand, q_dsl
    t_hand = timed(lambda: hand.quotient_values(lde, args.log_n, alpha), args.reps, args.warmup)
    t_dsl = timed(lambda: dsl.quotient_values(lde, args.log_n, alpha), args.reps, args.warmup)
    n_insn, slots, n_cons = dsl.program().info()
    lde_bytes = lde.numel() * 4
    print(json.dumps({"bench": "air_program_poseidon2", "gpu": name, "lde_rows": int(lde.shape[0]), "width": width, "instructions": n_insn,
                      "slots": slots, "constraints": n_cons, "hand_ms": round(t_hand, 3), "program_ms": round(t_dsl, 3),
                      "ratio": round(t_dsl / t_hand, 2), "program_trace_GBps": round(lde_bytes / t_dsl / 1e6, 1)}), flush=True)
    del lde


def mul_air(args, f, gpu, name, rng, alpha):
    # MulAir at 2^log_n rows, blowup 4, quotient domain 2^(log_n + 1)
    air = SymbolicAir(f, 60, E.mul_air_eval(3, True, True), gpu=gpu)
    trace = torch.from_numpy(rng.integers(0, f.P, (1 << args.log_n, 60), dtype=np.uint32).view(np.int32)).cuda()
    lde = gpu.coset_lde_batch(f.id, trace, 2, f.generator)
    qd = lde[: 2 << args.log_n]
    t = timed(lambda: air.quotient_values(qd, args.log_n, alpha), args.reps, args.warmup)
    n_insn, slots, n_cons = air.program().info()
    read = qd.numel() * 4 * 2                                        # local row + next row per quotient point
    print(json.dumps({"bench": "air_program_mul_air", "gpu": name, "trace_rows": 1 << args.log_n, "quotient_rows": int(qd.shape[0]),
                      "instructions": n_insn, "slots": slots, "constraints": n_cons, "ms": round(t, 3),
                      "trace_read_GBps": round(read / t / 1e6, 1)}), flush=True)


def mul_air_pre_eval(b):
    m, k, (u, v) = b.main(), b.preprocessed(), b.periodic_values()
    for i in range(E.REPETITIONS):
        a, bb, c = m.local[3 * i], m.local[3 * i + 1], m.local[3 * i + 2]
        b.assert_zero(a * a * bb * k.local[i] - c)
        b.when_first_row().assert_eq(a * a + 1, bb)
        b.when_transition().assert_eq(a + u + v, m.next[3 * i])


def mul_air_pre(args, f, gpu, name, rng, alpha):
    n = 1 << args.log_n
    pre = torch.from_numpy(rng.integers(0, f.P, (n, E.REPETITIONS), dtype=np.uint32).view(np.int32)).cuda()
    periodic = [[int(x) for x in rng.integers(0, f.P, 4)], [int(x) for x in rng.integers(0, f.P, 16)]]
    air = SymbolicAir(f, 60, mul_air_pre_eval, gpu=gpu, preprocessed_trace=pre, preprocessed_next_row_columns=[], periodic_columns=periodic)
    trace = torch.from_numpy(rng.integers(0, f.P, (n, 60), dtype=np.uint32).view(np.int32)).cuda()
    lde = gpu.coset_lde_batch(f.id, trace, 2, f.generator)
    pre_lde = gpu.coset_lde_batch(f.id, pre, 2, f.generator)
    qd, pq = lde[: 2 * n], pre_lde[: 2 * n]
    t = timed(lambda: air.quotient_values(qd, args.log_n, alpha, preprocessed_on_quotient_domain=pq), args.reps, args.warmup)
    n_insn, slots, n_cons = air.program().info()
    read = (qd.numel() * 2 + pq.numel()) * 4                          # main local + next rows, preprocessed local rows
    print(json.dumps({"bench": "air_program_mul_air_preprocessed_periodic", "gpu": name, "trace_rows": n, "quotient_rows": int(qd.shape[0]),
                      "preprocessed_width": E.REPETITIONS, "periods": [len(c) for c in periodic], "instructions": n_insn, "slots": slots,
                      "constraints": n_cons, "ms": round(t, 3), "trace_read_GBps": round(read / t / 1e6, 1)}), flush=True)


if __name__ == "__main__":
    main()
