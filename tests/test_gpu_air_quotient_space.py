"""The AIR quotient kernels over their launch space, each called through its C entry point and compared word for word with the
constraint-DAG oracle (tests/air_oracle.py) evaluated on the device:

    sweeps          SHA-256, Blake3 and Poseidon1 (vector_len 1, 8, 32) sized from the SM count so that the persistent blocks make at
                    least two full trips over the points plus a partial one, on valid-trace and uniformly random LDEs of both fields,
                    and once on an LDE taller than 2N (the quotient reads its prefix)
    vector lengths  Poseidon1 and both Poseidon2 instances at vector_len 1, 2, 4, 8, 16 and 32
    extremes        every hand-written kernel on LDEs of all Montgomery(p - 1), all zeros, rows alternating 0 and p - 1, and random
                    words, under the alphas (p - 1, p - 1, p - 1, p - 1), one and zero
    sharded         the SHA-256, Blake3 and Poseidon1 sharded kernels on every rank's chunk-major row block of a world-2 and a world-4
                    commit, laid out on one GPU, each rank's points spanning at least two sweeps
    rate bits       the constraint-program kernel on random DAGs at q = 4, 6 and 8 extra bits, up to 2^20 points

Every output goes into a buffer of 0xFFFFFFFF with guard rows on both sides: the guards must survive, every word must be below p and
equal the oracle's; a failure names the first differing natural index and the number of rows that differ."""
import ctypes as C

import numpy as np
import pytest
import torch

import air_oracle as A
import blake3_air_oracle as B3O
import keccak_air_oracle as KO
import poseidon1_air_oracle as PO
import poseidon2_babybear_air_oracle as BO
import sha256_air_oracle as SO
from oracle import p3_oracle as O
from plonky3_b200 import _lib
from plonky3_b200 import poseidon1_air as P1A
from plonky3_b200.blake3_air import Blake3Air
from plonky3_b200.distributed import block_view, chunk_major_block, column_starts, quotient_slice_natural_indices
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from plonky3_b200.poseidon2_air import RoundConstants, VectorizedPoseidon2Air
from plonky3_b200.sha256_air import Sha256Air
from test_air_program_cpu import random_dag

pytestmark = pytest.mark.gpu
FIELDS = [BabyBear, KoalaBear]
GUARD = 64                                     # EF4 rows of 0xFFFFFFFF on each side of every output
POISON = -1                                    # 0xFFFFFFFF as int32: above p in both fields

# Points per block of the persistent quotient kernels: hand_quotient_launch (air_program.cu) launches min(SMs, blocks) blocks, and each
# strides over the points by gridDim.x times this many.
SQ_POINTS = 24                                 # sha256_air.cu SQ_WARPS: one warp per point
BQ_POINTS = 16                                 # blake3_air.cu BQ_WARPS: one warp per point
P1Q_THREADS = 16 * 32                          # poseidon1_air.cu P1Q_WARPS warps, vector_len lanes per point


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sweep_log_points(per_block, world=1):
    """log2 of the smallest power-of-two quotient domain whose 1 / world share spans at least two full sweeps of min(SMs, blocks)
    persistent blocks plus a partial one; asserts it does, so that a device with more SMs cannot shrink the case."""
    sweep = _sms() * per_block
    log_pts = (2 * sweep * world).bit_length()
    while ((1 << log_pts) // world) % sweep == 0:
        log_pts += 1
    share = (1 << log_pts) // world
    assert share // sweep >= 2 and share % sweep, (share, sweep)
    return log_pts


def _monty(f, vals):
    return np.array([f.to_monty(int(v) % f.P) for v in vals], dtype=np.uint32)


def _random_alpha(f, seed):
    return _monty(f, np.random.default_rng(seed).integers(0, f.P, 4))


def _guarded(gpu, n, launch):
    """launch(output pointer) into n EF4 rows inside guard rows of 0xFFFFFFFF; returns the (n, 4) device view after checking the
    guards."""
    buf = torch.full((n + 2 * GUARD, 4), POISON, dtype=torch.int32, device="cuda")
    gpu._use_torch_stream()
    _lib.check(launch(buf[GUARD:GUARD + n].data_ptr()))
    torch.cuda.synchronize()
    assert bool((buf[:GUARD] == POISON).all()) and bool((buf[GUARD + n:] == POISON).all()), "write outside the quotient"
    return buf[GUARD:GUARD + n]


def _compare(f, got, exp, what, natural=None):
    """got, exp: (n, 4) int32 device tensors of u32 words; natural[m]: the natural index of row m (default m)."""
    words = got.to(torch.int64) & 0xFFFFFFFF
    above = torch.nonzero((words >= f.P).any(dim=1)).flatten()
    bad = torch.nonzero((got != exp).any(dim=1)).flatten()
    nat = (lambda m: int(natural[int(m)])) if natural is not None else int
    assert above.numel() == 0, f"{what}: natural index {nat(above[0])} holds a word >= p ({above.numel()} rows)"
    assert bad.numel() == 0, (f"{what}: natural index {nat(bad[0])}: got {got[bad[0]].tolist()} expected {exp[bad[0]].tolist()} "
                              f"({bad.numel()} rows differ)")


def _alpha_ptr(alpha):
    a = np.ascontiguousarray(alpha, dtype=np.uint32)
    return a, a.ctypes.data


# ---------------------------------------------------------------- the kernels and their DAGs
def _p2_constants(f):
    if f is BabyBear:
        return BO.example_constants()
    oair = O.air_from_rng(KoalaBear.id, O.SmallRng(1))          # the config-5 benchmark's constants
    return RoundConstants(np.array(oair.beg).reshape(4, 16), np.array(oair.part)[: oair.rounds_p], np.array(oair.end).reshape(4, 16))


_P2_DAGS = {}


def _kernel(gpu, name, f, vector_len=8):
    """(dag (nodes, constraints), width, quotient(lde, log_lde, log_n, alpha) -> the guarded output as a (points, 4) device tensor,
    log_points(log_lde, log_n)), after setting the AIR's constants on the context for this field."""
    L, h = gpu.L, gpu.h
    log_points = lambda log_lde, log_n: log_n + 1                 # the hand-written kernels' quotient domain: 2N points
    if name == "poseidon1":
        width = P1A.VectorizedPoseidon1Air(f, PO.optimized(f), gpu, vector_len=vector_len).width()
        dag, entry = PO.air_dag(f, vector_len), lambda *a: L.p3gpu_p1air_quotient_dev(h, f.id, vector_len, *a)
    elif name == "poseidon2":
        c = _p2_constants(f)
        VectorizedPoseidon2Air(f, c, gpu, vector_len=vector_len)
        if (f.id, vector_len) not in _P2_DAGS:
            air = VectorizedPoseidon2Air(f, c, None, vector_len=vector_len)
            _P2_DAGS[f.id, vector_len] = ((air.nodes, air.constraints), air.width())
        dag, width = _P2_DAGS[f.id, vector_len]
        entry = lambda *a: L.p3gpu_p2air_quotient_dev(h, f.id, vector_len, *a)
        log_points = lambda log_lde, log_n: log_lde                # the Poseidon2 kernel's: the whole LDE domain
    else:
        oracle, e, width = {"sha256": (SO, L.p3gpu_sha256_air_quotient_dev, _lib.SHA256_AIR_COLS),
                            "blake3": (B3O, L.p3gpu_blake3_air_quotient_dev, _lib.BLAKE3_AIR_COLS),
                            "keccak": (KO, L.p3gpu_keccak_air_quotient_dev, _lib.KECCAK_AIR_COLS)}[name]
        dag, entry = oracle.air_dag(f), lambda *a: e(h, f.id, *a)

    def quotient(lde, log_lde, log_n, alpha):
        al, ptr = _alpha_ptr(alpha)
        return _guarded(gpu, 1 << log_points(log_lde, log_n), lambda out: entry(lde.data_ptr(), log_lde, log_n, ptr, out))
    return dag, width, quotient, log_points


def _check(f, dag, lde, log_q, log_n, got, alphas, what):
    """got: one kernel output per alpha; one oracle evaluation for all of them."""
    exps = A.air_quotients(f.id, dag[0], dag[1], lde, log_q, log_n, [], alphas)
    for al, g, e in zip(alphas, got, exps):
        _compare(f, g, e, f"{what}, alpha {np.asarray(al).tolist()}")


def _random_lde(f, rows, width, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(0, f.P, (rows, width), dtype=torch.int32, device="cuda", generator=g)


def _valid_lde(gpu, name, f, log_n, log_blowup, seed, vector_len=8):
    """The coset LDE of a valid trace of 2^log_n rows, generated on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if name == "poseidon1":
        air = P1A.VectorizedPoseidon1Air(f, PO.optimized(f), gpu, vector_len=vector_len)
        inputs = torch.randint(0, f.P, (vector_len << log_n, 16), dtype=torch.int32, device="cuda", generator=g)
    else:
        air = (Sha256Air if name == "sha256" else Blake3Air)(f, gpu)
        inputs = torch.randint(-(1 << 31), 1 << 31, (1 << log_n, 24), dtype=torch.int32, device="cuda", generator=g)
    trace = air.generate_trace_rows(inputs)
    del inputs
    return gpu.coset_lde_batch(f.id, trace, log_blowup, f.generator, bitrev_rows=True)


# ---------------------------------------------------------------- sweeps
SWEEPS = [("sha256", 1, SQ_POINTS), ("blake3", 1, BQ_POINTS), ("poseidon1", 1, P1Q_THREADS // 1), ("poseidon1", 8, P1Q_THREADS // 8),
          ("poseidon1", 32, P1Q_THREADS // 32)]


@pytest.mark.parametrize("name,vector_len,per_block", SWEEPS, ids=[f"{s[0]}-v{s[1]}" for s in SWEEPS])
@pytest.mark.parametrize("f", FIELDS, ids=[f.name for f in FIELDS])
def test_past_the_first_persistent_sweep(gpu, f, name, vector_len, per_block):
    """At 132 SMs: 2^13 points for SHA-256 and Blake3, 2^18 / 2^15 / 2^13 for Poseidon1 at vector_len 1 / 8 / 32."""
    log_n = _sweep_log_points(per_block) - 1
    dag, width, quotient, _ = _kernel(gpu, name, f, vector_len)
    alpha = _random_alpha(f, log_n + 31 * vector_len)
    for kind, log_blowup in (("valid", 1), ("random", 2)):          # the random LDE is 4N rows tall: the quotient reads its prefix
        if kind == "valid":
            lde = _valid_lde(gpu, name, f, log_n, log_blowup, log_n + vector_len, vector_len)
        else:
            lde = _random_lde(f, 1 << (log_n + log_blowup), width, log_n)
        got = quotient(lde, log_n + log_blowup, log_n, alpha)
        _check(f, dag, lde, log_n + 1, log_n, [got], [alpha], f"{name} {f.name} {kind} 2^{log_n + 1} points of an LDE of 2^{log_n + log_blowup}")
        del lde, got
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- vector lengths
VECTOR_LENS = [1, 2, 4, 8, 16, 32]


@pytest.mark.parametrize("vector_len", VECTOR_LENS)
@pytest.mark.parametrize("name", ["poseidon1", "poseidon2"])
@pytest.mark.parametrize("f", FIELDS, ids=[f.name for f in FIELDS])
def test_every_vector_length(gpu, f, name, vector_len):
    """The lane count per point, the shuffle reduction over it, the padded alpha-table stride and the shared memory (BabyBear at 32:
    about 142 KB) all follow the vector length.  Poseidon2: BabyBear is the register instance, KoalaBear the config-5 kernel."""
    log_n = 7
    dag, width, quotient, points = _kernel(gpu, name, f, vector_len)
    lde = _random_lde(f, 2 << log_n, width, vector_len)
    alpha = _random_alpha(f, vector_len)
    got = quotient(lde, log_n + 1, log_n, alpha)
    _check(f, dag, lde, points(log_n + 1, log_n), log_n, [got], [alpha], f"{name} {f.name} vector_len {vector_len}")


# ---------------------------------------------------------------- value extremes
KERNELS = ["sha256", "blake3", "keccak", "poseidon1", "poseidon2"]
FILLS = ["p_minus_1", "zero", "alternating", "random"]


def _fill(f, kind, rows, width):
    top = f.to_monty(f.P - 1)
    if kind == "p_minus_1":
        return torch.full((rows, width), top, dtype=torch.int32, device="cuda")
    if kind == "zero":
        return torch.zeros((rows, width), dtype=torch.int32, device="cuda")
    if kind == "alternating":
        return (torch.arange(rows, device="cuda") % 2 * top).to(torch.int32).view(-1, 1).expand(rows, width).contiguous()
    return _random_lde(f, rows, width, 99)


@pytest.mark.parametrize("fill", FILLS)
@pytest.mark.parametrize("name", KERNELS)
@pytest.mark.parametrize("f", FIELDS, ids=[f.name for f in FIELDS])
def test_value_extremes(gpu, f, name, fill):
    """The lazy 64-bit accumulators (air_qmac) at their largest inputs and the folds at alphas whose powers are all p - 1 (up to
    sign), all the field's one, or zero past the last constraint.  The rows need not be a real LDE: kernel and oracle read whatever
    rows they are given."""
    log_n = 6
    dag, width, quotient, points = _kernel(gpu, name, f)
    lde = _fill(f, fill, 2 << log_n, width)
    alphas = [_monty(f, [f.P - 1] * 4), _monty(f, [1, 0, 0, 0]), _monty(f, [0, 0, 0, 0])]
    got = [quotient(lde, log_n + 1, log_n, al) for al in alphas]
    _check(f, dag, lde, points(log_n + 1, log_n), log_n, got, alphas, f"{name} {f.name} {fill}")


# ---------------------------------------------------------------- sharded instances on one GPU
SHARDED = [("sha256", 1, SQ_POINTS), ("blake3", 1, BQ_POINTS), ("poseidon1", 8, P1Q_THREADS // 8)]


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("name,vector_len,per_block", SHARDED, ids=[s[0] for s in SHARDED])
@pytest.mark.parametrize("f", FIELDS, ids=[f.name for f in FIELDS])
def test_sharded_blocks_past_the_first_sweep(gpu, f, name, vector_len, per_block, world):
    """Every rank's chunk-major row block of a world-2 / world-4 commit (distributed.chunk_major_block), each rank's points spanning
    at least two sweeps: at 132 SMs 2^14 / 2^15 points for SHA-256 and Blake3, 2^16 / 2^17 for Poseidon1.  The rank's slice, in
    bit-reversed order, against the oracle at quotient_slice_natural_indices."""
    log_q = _sweep_log_points(per_block, world)
    log_n = log_q - 1
    dag, width, _, _ = _kernel(gpu, name, f, vector_len)
    lde = _random_lde(f, 1 << log_q, width, log_q + world)
    alpha = _random_alpha(f, world + log_q)
    exp = A.air_quotient(f.id, dag[0], dag[1], lde, log_q, log_n, [], alpha)
    L, h = gpu.L, gpu.h
    entry = {"sha256": lambda *a: L.p3gpu_sha256_air_quotient_sharded_dev(h, f.id, *a),
             "blake3": lambda *a: L.p3gpu_blake3_air_quotient_sharded_dev(h, f.id, *a),
             "poseidon1": lambda *a: L.p3gpu_p1air_quotient_sharded_dev(h, f.id, vector_len, *a)}[name]
    R = (1 << log_q) // world
    starts = column_starts(width, world, align=8)
    cs = (C.c_size_t * len(starts))(*starts)
    al, ptr = _alpha_ptr(alpha)
    for rank in range(world):
        block = chunk_major_block(lde[rank * R:(rank + 1) * R], world, starts)
        st = block_view(world, rank, block)
        got = _guarded(gpu, R, lambda out: entry(C.byref(st), cs, log_q, log_n, ptr, out))
        nat = quotient_slice_natural_indices(rank, R, log_q)
        _compare(f, got, exp[torch.from_numpy(nat).cuda()], f"{name} {f.name} world {world} rank {rank}", natural=nat)
        del block, got


# ---------------------------------------------------------------- the constraint-program kernel at high rate bits
# (field, log_n, q, width, n_public, n_nodes, n_constraints)
RATES = [(BabyBear, 3, 4, 5, 2, 120, 12), (KoalaBear, 6, 6, 9, 1, 200, 20), (BabyBear, 4, 8, 3, 0, 80, 8), (KoalaBear, 12, 8, 6, 2, 150, 15)]


@pytest.mark.parametrize("case", RATES, ids=[f"{c[0].name}-n{c[1]}-q{c[2]}" for c in RATES])
def test_constraint_program_at_high_rate_bits(gpu, case):
    """Z_H and 1 / Z_H take 2^q values (tables of up to 256 entries at AIR_MAX_RATE_BITS = 8), indexed by i mod 2^q; the next row is
    2^q points on.  The matrix is a random bit-reversed one of 2^(log_n + q) rows, the last case 2^20 points."""
    f, log_n, q, width, n_public, n_nodes, n_cons = case
    rng = np.random.default_rng(log_n * 37 + q)
    nodes, cons = random_dag(f, rng, width, n_public, n_nodes, n_cons)
    log_q = log_n + q
    lde = _random_lde(f, 1 << log_q, width, log_q)
    pubs = _monty(f, rng.integers(0, f.P, n_public))
    alpha = _random_alpha(f, q)
    prog = gpu.air_program_create(f.id, nodes, cons, width, n_public)
    al, ptr = _alpha_ptr(alpha)
    got = _guarded(gpu, 1 << log_q, lambda out: gpu.L.p3gpu_air_quotient_dev(gpu.h, prog.h, lde.data_ptr(), log_q, log_q, log_n,
                                                                              pubs.ctypes.data if pubs.size else None, ptr, out))
    exp = A.air_quotient(f.id, nodes, cons, lde, log_q, log_n, [int(v) for v in pubs], alpha)
    _compare(f, got, exp, f"constraint program {f.name} 2^{log_q} points, q = {q}")
