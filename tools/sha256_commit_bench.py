"""Merkle commit of the config-3 shape (2^22 rows x 100 columns, BabyBear, one matrix) under both SHA-256 hash kinds against Keccak,
in one process, and the SHA-256 leaf kernel's compression rate against the integer-pipe floor of its SASS:

    python tools/sha256_commit_bench.py [--log-rows 22] [--width 100] [--reps 5]

Commit times are CUDA events around `Gpu.merkle_commit` (device-resident input), the three kinds alternating, median of --reps after
a warm-up.  Kernel times come from a separate torch.profiler run.  A 100-column row is 400 bytes, 7 SHA-256 blocks with the padding.

The floor: one compression is SHA256_ALU_INSTRS instructions on the ALU pipe (SHF, LOP3, IADD3; `cuobjdump -sass` of
sha256_compress_kernel<false>, sm_90a, which is one compression and the digest loads and stores), and an SM's ALU pipe takes 64 thread
instructions per clock (16 lanes per SM sub-partition), so compressions/s <= SMs * SM clock * 64 / SHA256_ALU_INSTRS at the card's
maximum SM clock.  Prints one JSON object with the card's name, power limit and maximum SM clock."""
import argparse
import json
import pathlib
import statistics
import subprocess
import sys

ROOT = pathlib.Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch

from plonky3_b200 import _lib
from plonky3_b200.field import BabyBear
from plonky3_b200.gpu import default_gpu

SHA256_ALU_INSTRS = 667 + 348 + 240          # SHF + LOP3 + IADD3 of one compression (its 114 IMADs issue on the FMA pipe)
ALU_LANES_PER_SM = 64


def _smi(q):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-rows", type=int, default=22)
    ap.add_argument("--width", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    gpu = default_gpu(0)
    n, w = 1 << a.log_rows, a.width
    g = torch.Generator(device="cuda"); g.manual_seed(3)
    x = torch.randint(0, BabyBear.P, (n, w), device="cuda", dtype=torch.int32, generator=g)
    kinds = {"sha256": _lib.HASH_SHA256, "sha256-compress": _lib.HASH_SHA256_COMPRESS, "keccak": _lib.HASH_KECCAK}
    times = {k: [] for k in kinds}
    for k in kinds.values():
        gpu.merkle_commit(BabyBear.id, k, [x])
    torch.cuda.synchronize()
    for _ in range(a.reps):
        for name, k in kinds.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(); gpu.merkle_commit(BabyBear.id, k, [x]); e.record(); e.synchronize()
            times[name].append(s.elapsed_time(e))
    # kernel times, in their own run
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in kinds.values():
            gpu.merkle_commit(BabyBear.id, k, [x])
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if any(t in ev.key for t in ("sha256_leaf", "sha256_compress", "keccak_leaf", "keccak_compress")):
            kern[ev.key] = {"launches": ev.count, "ms_per_launch": round(ev.device_time_total / 1e3 / max(ev.count, 1), 4)}
    leaf_ms = next((v["ms_per_launch"] for key, v in kern.items() if "sha256_leaf" in key), None)
    blocks = (4 * w + 9 + 63) // 64
    rate = n * blocks / (leaf_ms / 1e3) if leaf_ms else None
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clk = _smi("clocks.max.sm")
    floor = sms * float(clk) * 1e6 * ALU_LANES_PER_SM / SHA256_ALU_INSTRS if clk else None
    print(json.dumps({
        "card": _smi("name") or torch.cuda.get_device_name(0), "power_limit_w": _smi("power.limit"), "max_sm_clock_mhz": clk, "sms": sms,
        "shape": [n, w], "commit_ms_median": {k: round(statistics.median(v), 3) for k, v in times.items()},
        "commit_ms_all": {k: [round(t, 3) for t in v] for k, v in times.items()},
        "kernel_ms_profiler": kern, "sha256_blocks_per_row": blocks,
        "sha256_leaf_compressions_per_s": float("%.4g" % rate) if rate else None,
        "alu_pipe_floor_compressions_per_s": float("%.4g" % floor) if floor else None,
        "leaf_share_of_floor": round(rate / floor, 3) if rate and floor else None}))


if __name__ == "__main__":
    main()
