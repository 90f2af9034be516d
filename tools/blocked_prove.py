"""Prove the Blake3 and SHA-256 `-l 20` statements on one GPU with the LDE held as coefficients plus one coset
(coset_blocks.prove_coset_blocked), verify each proof, and compare with the resident-LDE `prove` at 2^19 rows.

The statements are tools/air_prove.py's (random inputs, one compression per row) under the Keccak configuration (cap height 3,
new_benchmark_high_arity's FRI parameters, log_blowup 1).  At 2^20 rows the trace and its whole LDE need 115 GB (Blake3, 9168 columns)
and 97 GB (SHA-256, 7728), more than an 80 GB card holds; the coset-blocked prove needs about twice the trace.  For each AIR it prints
one JSON line per run: prove ms per span, the total, torch.cuda.max_memory_allocated, the planned peak, and the card.  At 2^19 rows
both provers run, so the difference is the cost of recomputing the cosets (1 inverse DFT and 5 coset DFTs per prove at blowup 2,
against 1 + 2 with the LDE resident).

    python tools/blocked_prove.py [--air blake3 sha256] [--log-rows 20] [--field koala-bear]
"""
import argparse
import importlib.util
import json
import pathlib
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from plonky3_b200.coset_blocks import coset_blocked_memory_bytes, prove_coset_blocked  # noqa: E402
from plonky3_b200.dft import Radix2DitParallel  # noqa: E402
from plonky3_b200.field import BabyBear, KoalaBear  # noqa: E402
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs  # noqa: E402
from plonky3_b200.gpu import default_gpu  # noqa: E402
from plonky3_b200.merkle_tree import MerkleTreeMmcs  # noqa: E402
from plonky3_b200.uni_stark import KeccakStarkConfig, prove, verify  # noqa: E402


def _air_prove():
    spec = importlib.util.spec_from_file_location("air_prove", ROOT / "tools" / "air_prove.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def run(ap, air_name, f, gpu, config, log_rows, blocked):
    make, _, hashes, random_inputs, dtype = ap.AIRS[air_name]
    air = make(f, gpu)
    inputs = torch.from_numpy(np.ascontiguousarray(random_inputs(f, hashes(log_rows))).view(dtype)).cuda()
    trace = air.generate_trace_rows(inputs)
    del inputs
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    proof = prove_coset_blocked(config, air, trace) if blocked else prove(config, air, trace)
    torch.cuda.synchronize()
    total = (time.perf_counter() - t0) * 1e3
    peak = torch.cuda.max_memory_allocated()
    trace_bytes = trace.numel() * 4
    del trace
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    verify(config, air, proof)
    verify_ms = (time.perf_counter() - t0) * 1e3
    return {"air": air_name, "field": f.name, "log_rows": log_rows, "prover": "coset-blocked" if blocked else "prove",
            "prove_ms": round(total, 1), "spans_ms": {k: round(v, 1) for k, v in proof.timings_ms.items()},
            "max_memory_allocated": peak, "trace_bytes": trace_bytes,
            "planned_peak": coset_blocked_memory_bytes(air, log_rows, 1) if blocked else None,
            "proof_bytes": len(proof.to_postcard()), "verified": True, "verify_ms": round(verify_ms, 1)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--air", nargs="+", choices=["blake3", "sha256"], default=["blake3", "sha256"])
    p.add_argument("--log-rows", type=int, default=20)
    p.add_argument("--field", choices=["koala-bear", "baby-bear"], default="koala-bear")
    a = p.parse_args()
    f = KoalaBear if a.field == "koala-bear" else BabyBear
    gpu = default_gpu(0)
    m = MerkleTreeMmcs.keccak(f, cap_height=3, gpu=gpu)
    config = KeccakStarkConfig(TwoAdicFriPcs(Radix2DitParallel(f, gpu), m, FriParameters.new_benchmark_high_arity(m)))
    ap = _air_prove()
    card = _card()
    for air_name in a.air:
        for log_rows, blocked in [(a.log_rows, True), (a.log_rows - 1, True), (a.log_rows - 1, False)]:
            r = run(ap, air_name, f, gpu, config, log_rows, blocked)
            r["card"] = card
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
