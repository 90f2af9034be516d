"""The debug constraint check (air.check_all_constraints) of the hand-written AIRs at tools/air_prove.py's statements and shapes,
timed against `prove` of the same trace:

    python tools/air_check.py [--air keccak blake3 sha256 poseidon1 poseidon2] [--field koala-bear] [--log-rows N] [--reps 3]

Per AIR: the check program's size (instructions, slots, constraints), the check of the valid trace (both passes' host calls:
per-row counts, the device cumsum and row selection; median of --reps after a warm-up, host clock around work that ends in a device
synchronise), the same with one tampered cell (the report then lists its failures), and one `prove` under the Keccak
configuration after a warm-up.  Prints one JSON object per AIR with the card's name and power limit."""
import argparse
import importlib.util
import json
import pathlib
import statistics
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np
import torch

from plonky3_b200.air import check_all_constraints
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.uni_stark import KeccakStarkConfig, prove


def _air_prove():
    spec = importlib.util.spec_from_file_location("air_prove", ROOT / "tools" / "air_prove.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _timed(fn, reps):
    fn()
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out), r


def main():
    AP = _air_prove()
    ap = argparse.ArgumentParser()
    ap.add_argument("--air", nargs="+", choices=sorted(AP.AIRS), default=["keccak", "blake3", "sha256", "poseidon1", "poseidon2"])
    ap.add_argument("--field", choices=["koala-bear", "baby-bear"], default="koala-bear")
    ap.add_argument("--log-rows", type=int, default=None, help="trace height (default: tools/air_prove.py's for each AIR)")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    f = KoalaBear if a.field == "koala-bear" else BabyBear
    gpu = default_gpu(0)
    card = AP._card()
    for name in a.air:
        Air, default_log_rows, hashes, random_inputs, dtype = AP.AIRS[name]
        log_rows = default_log_rows if a.log_rows is None else a.log_rows
        air = Air(f, gpu)
        inputs = torch.from_numpy(np.ascontiguousarray(random_inputs(f, hashes(log_rows))).view(dtype)).cuda()
        trace = air.generate_trace_rows(inputs)
        del inputs
        n_insns, n_slots, n_cons = air.check_program().info()
        ok_ms, rep = _timed(lambda: check_all_constraints(air, trace), a.reps)
        assert rep.is_ok(), rep.failures[:5]
        row, col = (1 << log_rows) - 2, air.width() // 2
        keep = int(trace[row, col])
        trace[row, col] = (keep + 1) % f.P
        bad_ms, bad = _timed(lambda: check_all_constraints(air, trace), a.reps)
        assert not bad.is_ok() and {x.row for x in bad.failures} == {row}
        trace[row, col] = keep
        m = MerkleTreeMmcs.keccak(f, cap_height=3, gpu=gpu)
        config = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters.new_benchmark_high_arity(m)))
        prove(config, air, trace)
        prove_ms, _ = _timed(lambda: prove(config, air, trace), 1)
        rows = 1 << log_rows
        print(json.dumps({
            "air": name, "field": f.name, "card": card, "trace": [rows, air.width()],
            "check_program": {"instructions": n_insns, "slots": n_slots, "constraints": n_cons},
            "check_ms": round(ok_ms, 2), "check_tampered_ms": round(bad_ms, 2), "tampered_failures": len(bad.failures),
            "prove_ms": round(prove_ms, 2), "check_over_prove": round(ok_ms / prove_ms, 3),
            "instructions_per_s": float(f"{n_insns * rows / (ok_ms * 1e-3):.3e}"),
        }), flush=True)
        del trace, air, config
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
