"""`prove` of a hand-written-kernel AIR at the reference's `prove_prime_field_31` shapes, new_benchmark_high_arity's FRI parameters,
cap height 3.  One configuration per process:

    python tools/air_prove.py --air keccak --field koala-bear --config keccak [--log-rows 20] [--reps 3] [--kernel-reps 10]
    python tools/air_prove.py --air blake3 --field koala-bear --config keccak [--log-rows 18] [--reps 3] [--kernel-reps 10]
    python tools/air_prove.py --air sha256 --field koala-bear --config keccak [--log-rows 18] [--reps 3] [--kernel-reps 10]
    python tools/air_prove.py --air poseidon1 --field koala-bear --config keccak [--log-rows 20] [--reps 3] [--kernel-reps 10]
    python tools/air_prove.py --air poseidon2 --field baby-bear --config keccak [--log-rows 20] [--reps 3] [--kernel-reps 10]
    python tools/air_prove.py --air keccak --field baby-bear --config sha256 --fri benchmark --log-rows 15

  --config   keccak (Keccak MMCS, Keccak-256 transcript), poseidon2 (Poseidon2 MMCS, duplex transcript), sha256 / sha256-compress
             (SHA-256 MMCS with CompressionFunctionFromHasher<Sha256> or Sha256Compress nodes, SHA-256 transcript: the reference's
             prove_baby_bear_sha256 / _sha256_compress, whose KeccakAir statement is `--air keccak --fri benchmark --log-rows 15`)
  --fri      high-arity (new_benchmark_high_arity, the default) or benchmark (new_benchmark: arity 2)

  keccak   `-o keccak-f-permutations -l 20`: 43,690 hashes, a 2^20 x 2633 trace (the trace and its LDE take 33 GB together)
  blake3   `-o blake-3-permutations` at 2^18 compressions, a 2^18 x 9168 trace (29 GB with its LDE; the reference's `-l 20`
           shape, a 38.5 GB trace with a 77 GB LDE, does not fit on one 80 GB card)
  sha256   sha256-air's Sha256Air at 2^18 compressions, a 2^18 x 7728 trace (8.1 GB; its LDE 16.2 GB)
  poseidon1  `-o poseidon-1-permutations -l 20`: 8 << log_rows permutations, 8 per row, the constants of
           tests/golden/poseidon1_constants.json; a 2^20 x 1312 trace (KoalaBear, 5.5 GB) or 2^20 x 2384 (BabyBear, 10 GB)
  poseidon2  `-o poseidon-2-permutations -l 20`: 8 << log_rows permutations, 8 per row, the example's RoundConstants::from_rng on
           SmallRng(1) (13 partial rounds for BabyBear, 20 for KoalaBear); a 2^20 x 2384 trace (BabyBear, 10 GB) or 2^20 x 1312

Times trace generation and the quotient kernel alone (CUDA events, median of --kernel-reps launches after a warm-up), and `prove`
span by span (median of --reps proofs after one warm-up); then verifies the last proof.  Prints one JSON object with the card's name
and power limit, the quotient kernel's LDE bytes per second next to the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), named as
such, the peak device memory, and the SHA-256 of the last proof's bytes."""
import argparse
import hashlib
import json
import pathlib
import statistics
import subprocess
import sys
import time

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np
import torch

from plonky3_b200 import blake3_air, keccak_air, poseidon1_air, poseidon2_air, sha256_air
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import default_gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import KeccakStarkConfig, Sha256StarkConfig, StarkConfig, prove, verify

DATASHEET_HBM_BYTES_PER_S = 3.35e12          # NVIDIA H100 SXM data sheet, HBM3


def _poseidon1(f, gpu=None):
    """VectorizedPoseidon1Air with the fixture's constants (the example binary's), optimized as the reference does."""
    fx = json.loads((ROOT / "tests" / "golden" / "poseidon1_constants.json").read_text())[f.name]
    return poseidon1_air.VectorizedPoseidon1Air(f, poseidon1_air.Poseidon1Constants.from_fixture(f, fx).to_optimized(), gpu)


def _smallrng_inputs(f, n):
    """poseidon1_air.random_inputs(f, n), drawn by the C oracle of the same SmallRng: the scalar restatement takes minutes at
    2^23 permutations."""
    from oracle import p3_oracle as O
    return O.SmallRng(1).field(f.id, 16 * n).reshape(n, 16)


def _poseidon2(f, gpu=None):
    """VectorizedPoseidon2Air with the example binary's constants: RoundConstants::from_rng(SmallRng::seed_from_u64(1)), drawn by
    the C oracle of the same SmallRng."""
    from oracle import p3_oracle as O
    rp = 13 if f is BabyBear else 20
    c = O.air_from_rng(f.id, O.SmallRng(1), rp)
    consts = poseidon2_air.RoundConstants(np.array(c.beg, dtype=np.uint32).reshape(4, 16), np.array(c.part, dtype=np.uint32)[:rp],
                                          np.array(c.end, dtype=np.uint32).reshape(4, 16))
    return poseidon2_air.VectorizedPoseidon2Air(f, consts, gpu)


# --air: (AIR constructor (field, gpu), default --log-rows, hashes of a 2^log_rows trace, inputs (field, n), input dtype)
AIRS = {
    "keccak": (lambda f, gpu=None: keccak_air.KeccakAir(f, gpu), 20, lambda log_rows: (1 << log_rows) // 24,   # (24 n).next_power_of_two()
               lambda f, n: keccak_air.random_inputs(n), np.int64),
    "blake3": (lambda f, gpu=None: blake3_air.Blake3Air(f, gpu), 18, lambda log_rows: 1 << log_rows,           # one compression per row
               lambda f, n: blake3_air.random_inputs(n), np.int32),
    "sha256": (lambda f, gpu=None: sha256_air.Sha256Air(f, gpu), 18, lambda log_rows: 1 << log_rows,         # one compression per row
               lambda f, n: sha256_air.random_inputs(n), np.int32),
    "poseidon1": (_poseidon1, 20, lambda log_rows: 8 << log_rows, _smallrng_inputs, np.int32),               # 8 permutations per row
    "poseidon2": (_poseidon2, 20, lambda log_rows: 8 << log_rows, _smallrng_inputs, np.int32),               # the same SmallRng(1) draw
}


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def _events_median(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); e.synchronize()
        times.append(s.elapsed_time(e))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--air", choices=sorted(AIRS), required=True)
    ap.add_argument("--field", choices=["koala-bear", "baby-bear"], default="koala-bear")
    ap.add_argument("--config", choices=["keccak", "poseidon2", "sha256", "sha256-compress"], default="keccak")
    ap.add_argument("--fri", choices=["high-arity", "benchmark"], default="high-arity")
    ap.add_argument("--log-rows", type=int, default=None, help="trace height (default: 20 for keccak and poseidon1/2, 18 for blake3 and sha256)")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--kernel-reps", type=int, default=10)
    a = ap.parse_args()
    Air, default_log_rows, hashes, random_inputs, dtype = AIRS[a.air]
    log_rows = default_log_rows if a.log_rows is None else a.log_rows
    f = KoalaBear if a.field == "koala-bear" else BabyBear
    gpu = default_gpu(0)
    fri = FriParameters.new_benchmark if a.fri == "benchmark" else FriParameters.new_benchmark_high_arity
    if a.config == "keccak":
        m = MerkleTreeMmcs.keccak(f, cap_height=3, gpu=gpu)
        config = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, fri(m)))
    elif a.config in ("sha256", "sha256-compress"):
        m = MerkleTreeMmcs.sha256(f, cap_height=3, gpu=gpu, node="compress" if a.config == "sha256-compress" else "hasher")
        config = Sha256StarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, fri(m)))
    else:
        p16, p24 = default_poseidon2(f, 16), default_poseidon2(f, 24)
        m = MerkleTreeMmcs.poseidon2(p16, p24, cap_height=3, gpu=gpu)
        config = StarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, fri(m)), p24, 16)
    air = Air(f, gpu)
    n = hashes(log_rows)
    inputs = torch.from_numpy(random_inputs(f, n).view(dtype)).cuda()
    trace = air.generate_trace_rows(inputs)
    assert tuple(trace.shape) == (1 << log_rows, air.width())
    gen_ms = _events_median(lambda: air.generate_trace_rows(inputs), a.kernel_reps)
    trace_bytes = trace.numel() * 4

    # the quotient kernel alone, on the committed LDE's quotient-domain prefix (2^(log_rows + 1) rows)
    lde = gpu.coset_lde_batch(f.id, trace, 1, f.generator, bitrev_rows=True)
    alpha = np.array([f.to_monty(v) for v in (3, 5, 7, 11)], dtype=np.uint32)
    q_ms = _events_median(lambda: air.quotient_values(lde, log_rows, alpha), a.kernel_reps)
    lde_bytes = lde.numel() * 4
    del lde
    torch.cuda.empty_cache()

    prove(config, air, trace)                                    # warm-up: twiddles, constants, allocator
    spans, totals = {}, []
    for _ in range(a.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        proof = prove(config, air, trace)
        torch.cuda.synchronize()
        totals.append((time.perf_counter() - t0) * 1e3)
        for s, v in proof.timings_ms.items():
            spans.setdefault(s, []).append(v)
    raw = proof.to_postcard()
    del trace
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    verify(config, Air(f), raw)
    verify_ms = (time.perf_counter() - t0) * 1e3
    print(json.dumps({
        "card_and_power_limit": _card(), "air": a.air, "field": a.field, "config": a.config, "fri": a.fri, "hashes": n, "trace_rows": 1 << log_rows,
        "width": air.width(), "trace_generation_ms": round(gen_ms, 3), "trace_bytes_written": trace_bytes,
        "trace_generation_bytes_per_s": float("%.3g" % (trace_bytes / gen_ms * 1e3)),
        "quotient_kernel_ms": round(q_ms, 3), "quotient_lde_bytes_read": lde_bytes,
        "quotient_bytes_per_s": float("%.3g" % (lde_bytes / q_ms * 1e3)),
        "datasheet_hbm_bytes_per_s": DATASHEET_HBM_BYTES_PER_S,
        "prove_ms": round(statistics.median(totals), 1), "prove_spans_ms": {s: round(statistics.median(v), 2) for s, v in spans.items()},
        "peak_allocated_bytes": torch.cuda.max_memory_allocated(),
        "proof_bytes": len(raw), "proof_sha256": hashlib.sha256(raw).hexdigest(), "verify_ms": round(verify_ms, 1), "verified": True}))


if __name__ == "__main__":
    main()
