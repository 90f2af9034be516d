"""Per-CTA phase timeline of the NTT pass kernel (needs the instrumented build:
   P3GPU_OUT=$PWD/build/libp3gpu_prof.so P3GPU_OBJ=$PWD/build/obj_prof plonky3_b200/csrc/build.sh -DP3GPU_NTT_PROFILE
   P3GPU_LIB=$PWD/build/libp3gpu_prof.so python tools/ntt_timeline.py [w]).
Prints, per launch of one 2^20 x w LDE, the mean duration (us) of: cp.async issue, load wait, step 1, step 2 (+stores), and
the gap between a CTA's tiles.  The cp.async LDE is three launches: inverse layers 0-9, the fused pass (inverse layers 10-19 +
forward layers 0-9 of every coset; its "step1" is inverse step 1 and its "step2" all the rest) and forward layers 10-19; the
pipeline (P3GPU_NTT_PIPE=1) is four.  The first two store their tiles with tensor copies: their gap between tiles includes the
wait for the previous tile's store to leave the buffer that is refilled next, and the fused pass also reports the time it waits
for one coset's store before the next coset rewrites the tile buffer."""
import os, sys, pathlib
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
import torch
import numpy as np

w = int(sys.argv[1]) if len(sys.argv) > 1 else 100
buf = torch.zeros(8 * (1 << 17), dtype=torch.int64, device="cuda")
os.environ["P3GPU_NTT_PROFBUF"] = str(buf.data_ptr())
from plonky3_b200.field import KoalaBear as KB
from plonky3_b200.gpu import default_gpu
gpu = default_gpu(0)
x = torch.randint(0, KB.P, (1 << 20, w), device="cuda", dtype=torch.int32)
for _ in range(2):   # the launches of 2 LDEs take the 8 windows in turn; the second LDE is the warm one
    y = gpu.coset_lde_batch(KB.id, x, 1, KB.generator)
torch.cuda.synchronize()
raw = buf.cpu().numpy().reshape(8, -1)
names = ["inverse 0-9", "inverse 10-19", "forward 0-9", "forward 10-19"]
if os.environ.get("P3GPU_NTT_PIPE") == "1":   # dense LDEs take the cp.async kernel unless the pipeline is forced
    # pipelined kernel: slots per (CTA, group, tile): smid/unused, t_start, t_full, t_step1, t_step2
    for li in range(4, 8):
        d = raw[li].reshape(-1, 16, 8)
        rows = d[d[:, :, 4] != 0].astype(np.float64)
        print(f"launch {names[li - 4]}: {len(rows)} stamped group-tiles")
        print(f"   wait for tile {np.mean(rows[:, 2] - rows[:, 1]) / 1e3:6.2f} us (p50 {np.percentile(rows[:, 2] - rows[:, 1], 50) / 1e3:.2f}, p90 "
              f"{np.percentile(rows[:, 2] - rows[:, 1], 90) / 1e3:.2f}) | step1 {np.mean(rows[:, 3] - rows[:, 2]) / 1e3:6.2f} | "
              f"step2+stores {np.mean(rows[:, 4] - rows[:, 3]) / 1e3:6.2f} | total {np.mean(rows[:, 4] - rows[:, 1]) / 1e3:6.2f}")
    sys.exit(0)
b = raw.reshape(8, -1, 16, 8)
names = ["inverse 0-9", "inverse 10-19 + forward 0-9 (fused)", "forward 10-19"]
for li in range(3, 6):
    d = b[li]
    valid = d[:, :, 5] != 0
    n_cta = int(valid[:, 0].sum())
    rows = d[valid]
    start, issued, loaded, s1, s2 = (rows[:, i].astype(np.float64) for i in (1, 2, 3, 4, 5))
    print(f"launch {names[li - 3]}: {n_cta} CTAs, {len(rows)} stamped tiles")
    print(f"   issue {np.mean(issued - start) / 1e3:7.2f} us | load wait {np.mean(loaded - issued) / 1e3:7.2f} | step1 {np.mean(s1 - loaded) / 1e3:7.2f} | "
          f"step2+stores {np.mean(s2 - s1) / 1e3:7.2f} | tile total {np.mean(s2 - start) / 1e3:7.2f}")
    if li == 4:
        # slot 6: the waits for a coset's store to leave the tile buffer, summed over the tile's cosets (producer-warp form: the
        # producer's read-out waits, off the consumers' path); slot 7 (producer-warp form only): the consumers' waits for the
        # producer's `freed` before the next coset, and slot 2 is the producer's load issue
        print(f"   wait for the stores to be read out {np.mean(rows[:, 6].astype(np.float64)) / 1e3:7.2f} us per tile")
        if rows[:, 7].any():
            print(f"   consumers' wait for the buffer between cosets {np.mean(rows[:, 7].astype(np.float64)) / 1e3:7.2f} us per tile")
    # per CTA: gap between consecutive tiles (the wait for the store of the buffer refilled next, and the leading barrier)
    gaps = []
    for c in range(d.shape[0]):
        k = int(valid[c].sum())
        for j in range(1, k):
            gaps.append(float(d[c, j, 1]) - float(d[c, j - 1, 5]))
    if gaps:
        print(f"   gap between tiles {np.mean(gaps) / 1e3:6.2f} us; percentiles of load wait: "
              + ", ".join(f"p{q}={np.percentile(loaded - issued, q) / 1e3:.2f}" for q in (10, 50, 90)))
    t0 = rows[:, 1].min()
    span = (rows[:, 5].max() - t0) / 1e3
    print(f"   stamped span {span:.1f} us")
