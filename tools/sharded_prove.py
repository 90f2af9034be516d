"""Time distributed.prove_sharded against uni_stark.prove on the config-5 statement (2^L rows x 1312 KoalaBear columns, Poseidon2 AIR,
new_benchmark_high_arity, cap_height 3) in the same run, and assert that both write the same proof bytes.

    python tools/sharded_prove.py [L] [reps]                             one GPU, world = 1 (the cost of the sharded machinery)
    torchrun --nproc_per_node G tools/sharded_prove.py [L] [reps]        one process per GPU, world = G

Rank 0 prints one JSON line: card name, power limit, SM count, world, the per-span times of `prove` (rank 0) and of
`prove_sharded` (max over ranks), each the median over `reps` runs after one warm-up run."""
import json
import os
import pathlib
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))
from plonky3_b200.dft import Radix2DitParallel
from plonky3_b200.distributed import PeerGroup, column_starts, prove_sharded
from plonky3_b200.field import KoalaBear as KB
from plonky3_b200.fri import FriParameters, TwoAdicFriPcs
from plonky3_b200.gpu import Gpu
from plonky3_b200.merkle_tree import MerkleTreeMmcs
from plonky3_b200.poseidon2 import default_poseidon2
from plonky3_b200.uni_stark import RoundConstants, StarkConfig, VectorizedPoseidon2Air, prove

L = int(sys.argv[1]) if len(sys.argv) > 1 else 20
REPS = int(sys.argv[2]) if len(sys.argv) > 2 else 3
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
device = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(device)
if world > 1:
    import torch.distributed as dist
    dist.init_process_group("gloo")
gpu = Gpu(device)
mm = MerkleTreeMmcs.poseidon2(default_poseidon2(KB, 16), default_poseidon2(KB, 24), 3, gpu)
cfg = StarkConfig(TwoAdicFriPcs(Radix2DitParallel(KB, gpu), mm, FriParameters.new_benchmark_high_arity(mm)), default_poseidon2(KB, 24), 16)
rs = np.random.default_rng(7)
air = VectorizedPoseidon2Air(KB, RoundConstants(rs.integers(0, KB.P, (4, 16), dtype=np.uint32), rs.integers(0, KB.P, 20, dtype=np.uint32),
                                                rs.integers(0, KB.P, (4, 16), dtype=np.uint32)), gpu)
gen = torch.Generator(device=f"cuda:{device}"); gen.manual_seed(11)
inputs = torch.randint(0, KB.P, (8 << L, 16), device=f"cuda:{device}", dtype=torch.int32, generator=gen)   # same on every rank
W = air.width()


def median_spans(runs):
    return {k: float(np.median([r[k] for r in runs])) for k in runs[0]}


# single-GPU reference (every rank computes it; rank 0's times are reported)
trace = air.generate_trace_rows(inputs)
ref_runs = []
for i in range(REPS + 1):
    p = prove(cfg, air, trace)
    if i:
        ref_runs.append(dict(p.timings_ms, total=sum(p.timings_ms.values())))
expected = p.to_postcard()
del trace, p
torch.cuda.empty_cache()

starts = column_starts(W, world, align=8)
block = air.generate_trace_cols(inputs, starts[rank], starts[rank + 1])
grp = PeerGroup(gpu, (2 << L) // world, W, timeout_s=120.0)
sh_runs = []
for i in range(REPS + 1):
    p = prove_sharded(cfg, air, grp, block, starts)
    assert p.to_postcard() == expected, "prove_sharded wrote different proof bytes"
    if i:
        sh_runs.append(dict(p.timings_ms, total=sum(p.timings_ms.values())))
grp.close()

if rank == 0:
    q = subprocess.run(["nvidia-smi", f"--id={device}", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print(json.dumps({"card": q.stdout.strip(), "sm_count": torch.cuda.get_device_properties(device).multi_processor_count, "world": world,
                      "log_n": L, "width": W, "reps": REPS, "bytes_equal": True, "prove_ms": median_spans(ref_runs),
                      "prove_sharded_ms_max_over_ranks": median_spans(sh_runs)}))
if world > 1:
    dist.barrier()
    dist.destroy_process_group()
