"""Config-5 `prove` (the vectorised Poseidon2 AIR, KoalaBear, new_benchmark_high_arity, cap height 3) under the Keccak configuration
(Keccak MMCS, SerializingChallenger32 over Keccak-256) next to the Poseidon2 configuration, in one process, span by span.

    python tools/keccak_prove.py [--log-perms 20] [--reps 3] [--grind-bits 16 20 24]

Prints one JSON object: per configuration the median of each prove span (ms) over --reps proofs after one warm-up, the proof size,
and the grinding kernel's rate (candidates per second, from the number of candidates a grind had to test)."""
import argparse
import json
import pathlib
import statistics
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np
import torch

from plonky3_b200.challenger import SerializingChallenger32
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import KoalaBear as F
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import KeccakStarkConfig, RoundConstants, StarkConfig, VectorizedPoseidon2Air, prove


def _air(gpu):
    rng = np.random.default_rng(1)
    c = RoundConstants(F.to_monty_array(rng.integers(0, F.P, (4, 16), dtype=np.uint32)),
                       F.to_monty_array(rng.integers(0, F.P, 20, dtype=np.uint32)),
                       F.to_monty_array(rng.integers(0, F.P, (4, 16), dtype=np.uint32)))
    return VectorizedPoseidon2Air(F, c, gpu)


def _grind_rate(gpu, bits: int, trials: int):
    """Candidates tested per second: a grind from 0 tests (smallest witness + 1) candidates, rounded up to the launch batch."""
    rates = []
    for t in range(trials):
        ch = SerializingChallenger32.from_hasher([], F, gpu)
        ch.observe_slice(np.arange(t, t + 50, dtype=np.uint32))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w = ch.grind(bits)
        dt = time.perf_counter() - t0
        batch = 1 << min(22, bits + 3)
        tested = ((F.from_monty(w) // batch) + 1) * batch
        rates.append(tested / dt)
    return statistics.median(rates)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-perms", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--grind-bits", type=int, nargs="*", default=[16, 20, 24])
    a = ap.parse_args()
    gpu = default_gpu(0)
    p16, p24 = default_poseidon2(F, 16), default_poseidon2(F, 24)
    air = _air(gpu)
    inputs = torch.randint(0, F.P, (1 << a.log_perms, 16), device="cuda", dtype=torch.int32, generator=torch.Generator(device="cuda").manual_seed(1))
    trace = air.generate_trace_rows(inputs)
    configs = {}
    m = MerkleTreeMmcs.poseidon2(p16, p24, cap_height=3, gpu=gpu)
    configs["poseidon2"] = StarkConfig(TwoAdicFriPcs(Radix2DitParallel(F, gpu), m, FriParameters.new_benchmark_high_arity(m)), p24, 16)
    k = MerkleTreeMmcs.keccak(F, cap_height=3, gpu=gpu)
    configs["keccak"] = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(F, gpu), k, FriParameters.new_benchmark_high_arity(k)))
    out = {"log_perms": a.log_perms, "gpu": torch.cuda.get_device_name(0), "configs": {}}
    for name, cfg in configs.items():
        prove(cfg, air, trace)                                                    # warm-up: twiddles, constants, allocator
        spans, totals, size = {}, [], 0
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            proof = prove(cfg, air, trace)
            torch.cuda.synchronize()
            totals.append((time.perf_counter() - t0) * 1e3)
            for s, v in proof.timings_ms.items():
                spans.setdefault(s, []).append(v)
            size = len(proof.to_postcard())
        out["configs"][name] = {"prove_ms": round(statistics.median(totals), 2), "proof_bytes": size,
                                "spans_ms": {s: round(statistics.median(v), 2) for s, v in spans.items()}}
    out["keccak_grind_candidates_per_s"] = {str(b): float("%.3g" % _grind_rate(gpu, b, 5 if b < 24 else 2)) for b in a.grind_bits}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
