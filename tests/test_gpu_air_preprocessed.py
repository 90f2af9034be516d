"""Preprocessed and periodic columns on the GPU: p3gpu_air_quotient_layout_dev equals the oracle (tests/air_layout_oracle.py, periodic
columns evaluated directly) on poisoned, guarded buffers over both fields, trace heights 2^3 to 2^20, q = 0..3, preprocessed widths up to
~500 with and without the next row, periods 1 to n and a program near the slot limit; the new entry points refuse bad input before
anything launches; MulFibPAir, PeriodicAir and an AIR with both kinds prove on the GPU with the bytes of the same driver on the
oracle-backed stand-in device and are accepted by both verifiers; and setup_preprocessed's data serves two proofs."""
import numpy as np
import pytest
import torch

import air_layout_oracle as AL
import air_preprocessed_examples as X
from plonky3_b200 import _lib
from plonky3_b200.air import ADD, MAIN_LOCAL, MUL, PERIODIC, PREPROCESSED_LOCAL, PREPROCESSED_NEXT, SymbolicAir
from plonky3_b200.field import BabyBear, KoalaBear
from plonky3_b200.gpu import default_gpu
from test_air_preprocessed_cpu import ROUND_TRIPS, LayoutMockGpu, _air_and_trace, _config, random_layout_dag

pytestmark = pytest.mark.gpu
GUARD = 64
POISON = np.uint32(0xFFFFFFFF)


@pytest.fixture(scope="module")
def gpu():
    assert torch.cuda.is_available() and _lib.LIB_PATH.exists()
    return default_gpu(0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint32).view(np.int32)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint32)


def _guarded(gpu, prog, lde, pre, table, log_q, log_n, pubs, alpha):
    buf = dev(np.full(((1 << log_q) + 2 * GUARD, 4), POISON, dtype=np.uint32))
    out = buf[GUARD:GUARD + (1 << log_q)]
    gpu._use_torch_stream()
    pv = np.ascontiguousarray(pubs, dtype=np.uint32)
    lg = lambda t: int(t.shape[0]).bit_length() - 1
    _lib.check(gpu.L.p3gpu_air_quotient_layout_dev(gpu.h, prog.h, lde.data_ptr(), lg(lde), pre.data_ptr() if pre is not None else None,
                                                   lg(pre) if pre is not None else 0, table.data_ptr() if table is not None else None,
                                                   lg(table) if table is not None else 0, log_q, log_n, pv.ctypes.data if pv.size else None,
                                                   np.ascontiguousarray(alpha, dtype=np.uint32).ctypes.data, out.data_ptr()))
    b = host(buf)
    assert (b[:GUARD] == POISON).all() and (b[GUARD + (1 << log_q):] == POISON).all(), "write outside the quotient"
    return b[GUARD:GUARD + (1 << log_q)]


def _compare(got, exp):
    bad = np.flatnonzero((got != exp).any(axis=1))
    assert bad.size == 0, f"row {bad[0]}: got {got[bad[0]].tolist()} expected {exp[bad[0]].tolist()} ({bad.size} rows differ)"


def _check(gpu, f, nodes, cons, width, n_public, pre_width, periods, log_n, q, log_blowup, seed):
    rng = np.random.default_rng(seed)
    rand = lambda shape: f.to_monty_array(rng.integers(0, f.P, shape).astype(np.uint64)).astype(np.uint32)
    lde = gpu.coset_lde_batch(f.id, dev(rand((1 << log_n, width))), log_blowup, f.generator)
    pre = gpu.coset_lde_batch(f.id, dev(rand((1 << log_n, pre_width))), log_blowup, f.generator) if pre_width else None
    cols = [[int(v) for v in rng.integers(0, f.P, p)] for p in periods]
    pubs = [f.to_monty(int(v)) for v in rng.integers(0, f.P, n_public)]
    alpha = rand(4)
    air = SymbolicAir(f, width, lambda b: None, num_public_values=n_public, gpu=gpu, periodic_columns=cols,
                      preprocessed_trace=np.zeros((1 << log_n, pre_width), dtype=np.uint32) if pre_width else None)
    log_q = log_n + q
    table = air.periodic_table(log_n, log_q)
    prog = gpu.air_program_create_layout(f.id, nodes, cons, (width, n_public, pre_width, len(periods)))
    got = _guarded(gpu, prog, lde, pre, table, log_q, log_n, pubs, alpha)
    _compare(got, AL.air_quotient(f.id, nodes, cons, host(lde), log_q, log_n, pubs, alpha,
                                   pre_lde_bitrev=host(pre) if pre is not None else None, periodic_columns=cols))
    return prog


# (field, log_n, q, log_blowup, width, n_public, pre_width, periods, n_nodes, n_constraints)
RANDOM = [(BabyBear, 3, 0, 1, 2, 1, 1, [1], 40, 4), (KoalaBear, 3, 3, 3, 3, 0, 2, [8, 2], 60, 6),
          (BabyBear, 6, 1, 2, 5, 2, 9, [64, 4, 1], 150, 12), (KoalaBear, 8, 2, 2, 7, 0, 40, [256, 16], 300, 25),
          (BabyBear, 12, 1, 1, 16, 1, 500, [2, 32], 900, 60), (KoalaBear, 16, 2, 2, 4, 0, 3, [1024, 8], 120, 10),
          (BabyBear, 20, 1, 1, 2, 0, 2, [4, 16], 60, 5), (KoalaBear, 19, 0, 1, 3, 1, 1, [2], 40, 4)]


@pytest.mark.parametrize("case", RANDOM, ids=[f"{c[0].name}-n{c[1]}-q{c[2]}-pre{c[6]}-p{max(c[7])}" for c in RANDOM])
def test_random_layout_programs_match_oracle(gpu, case):
    f, log_n, q, lb, width, n_public, pre_width, periods, n_nodes, n_cons = case
    nodes, cons = random_layout_dag(f, np.random.default_rng(log_n * 7 + pre_width), width, n_public, pre_width, len(periods), n_nodes, n_cons)
    _check(gpu, f, nodes, cons, width, n_public, pre_width, periods, log_n, q, lb, seed=log_n + q)


@pytest.mark.parametrize("f", [BabyBear, KoalaBear])
def test_preprocessed_local_only_and_every_period(gpu, f):
    """Preprocessed columns read on the current row only (no next-row pointer), and periods 1, 2, ..., n of one trace."""
    log_n = 5
    periods = [1 << k for k in range(log_n + 1)]
    nodes = [(PREPROCESSED_LOCAL, c, 0, 0) for c in range(3)] + [(PERIODIC, k, 0, 0) for k in range(len(periods))]
    nodes += [(MAIN_LOCAL, 0, 0, 0)]
    acc = len(nodes) - 1
    for i in range(len(nodes) - 1):
        nodes.append((MUL, acc, i, 0)); nodes.append((ADD, len(nodes) - 1, i, 0)); acc = len(nodes) - 1
    cons = list(range(len(nodes) - 2 * (len(nodes) // 3), len(nodes)))
    for q, lb in ((0, 1), (1, 1), (2, 3), (3, 3)):
        _check(gpu, f, np.array(nodes), cons, 1, 0, 3, periods, log_n, q, lb, seed=q)


def test_program_near_the_slot_limit(gpu):
    """380 values live at once, from main, preprocessed (both rows) and periodic leaves."""
    f, width = KoalaBear, 190
    nodes = [(MAIN_LOCAL, c, 0, 0) for c in range(width)] + [(PREPROCESSED_NEXT, c, 0, 0) for c in range(width)]
    nodes += [(MUL, c, width + c, 0) for c in range(width)]
    nodes += [(PREPROCESSED_LOCAL, c, 0, 0) for c in range(width)] + [(PERIODIC, c % 3, 0, 0) for c in range(width)]
    nodes += [(MUL, 3 * width + c, 4 * width + c, 0) for c in range(width)]
    prods = list(range(2 * width, 3 * width)) + list(range(5 * width, 6 * width))
    acc = prods[0]
    for c in prods[1:]:
        nodes.append((ADD, acc, c, 0)); acc = len(nodes) - 1
    prog = _check(gpu, f, np.array(nodes), [acc] + prods, width, 0, width, [4, 2, 8], 6, 1, 1, seed=5)
    assert 380 <= prog.info()[1] <= 384


def test_one_row_periodic_table(gpu):
    """p_max = 1: the table is the LDE of a one-row matrix, a constant on every row."""
    f = BabyBear
    air = SymbolicAir(f, 1, lambda b: None, gpu=gpu, periodic_columns=[[7], [9]])
    for log_n, log_q in ((3, 3), (4, 6)):
        t = host(air.periodic_table(log_n, log_q))
        assert t.shape == (1 << (log_q - log_n), 2)
        assert (t[:, 0] == f.to_monty(7)).all() and (t[:, 1] == f.to_monty(9)).all()


# ---------------------------------------------------------------- bad input, refused before anything launches
def test_layout_entry_points_refuse_bad_input(gpu):
    f = KoalaBear
    nodes = [(MAIN_LOCAL, 0, 0, 0), (PREPROCESSED_LOCAL, 0, 0, 0), (PERIODIC, 0, 0, 0), (MUL, 0, 1, 0), (MUL, 3, 2, 0)]
    prog = gpu.air_program_create_layout(f.id, nodes, [4], (1, 0, 1, 1))
    lde = gpu.coset_lde_batch(f.id, dev(np.ones((16, 1), dtype=np.uint32)), 1, f.generator)       # 2^5 rows
    pre = gpu.coset_lde_batch(f.id, dev(np.ones((16, 1), dtype=np.uint32)), 1, f.generator)
    table = dev(np.ones((4, 1), dtype=np.uint32))
    alpha = np.zeros(4, dtype=np.uint32)
    gpu.air_quotient_layout(prog, lde, pre, table, 5, 4, [], alpha)                                 # well formed
    torch.cuda.synchronize()
    n0 = gpu.launches
    bad = [
        (lambda: gpu.air_quotient_layout(prog, lde, pre[:16], table, 5, 4, [], alpha), "preprocessed LDE of 2^4"),
        (lambda: gpu.air_quotient_layout(prog, lde, None, table, 5, 4, [], alpha), "preprocessed LDE missing"),
        (lambda: gpu.air_quotient_layout(prog, lde, pre, None, 5, 4, [], alpha), "periodic table missing"),
        (lambda: gpu.air_quotient_layout(prog, lde, pre, dev(np.ones((64, 1), dtype=np.uint32)), 5, 4, [], alpha), "periodic table of 2^6"),
        (lambda: gpu.air_quotient(prog, lde, 5, 4, [], alpha), "p3gpu_air_quotient_layout_dev"),     # the old entry point
    ]
    for call, msg in bad:
        with pytest.raises(_lib.P3GpuError) as ex:
            call()
        assert ex.value.code == _lib.EINVAL and msg in str(ex.value), str(ex.value)
    # a misaligned buffer
    flat = dev(np.ones(32 * 1 + 1, dtype=np.uint32))
    with pytest.raises(_lib.P3GpuError) as ex:
        _lib.check(gpu.L.p3gpu_air_quotient_layout_dev(gpu.h, prog.h, lde.data_ptr(), 5, flat.data_ptr() + 2, 5, table.data_ptr(), 2, 5, 4,
                                                       None, alpha.ctypes.data, dev(np.zeros((32, 4), dtype=np.uint32)).data_ptr()))
    assert ex.value.code == _lib.EINVAL and "misaligned" in str(ex.value)
    # a layout program without preprocessed columns given a preprocessed LDE
    prog2 = gpu.air_program_create_layout(f.id, [(PERIODIC, 0, 0, 0)], [0], (1, 0, 0, 1))
    with pytest.raises(_lib.P3GpuError) as ex:
        gpu.air_quotient_layout(prog2, lde, pre, table, 5, 4, [], alpha)
    assert ex.value.code == _lib.EINVAL
    with pytest.raises(_lib.P3GpuError) as ex:                                                       # out-of-range leaves
        gpu.air_program_create_layout(f.id, [(PREPROCESSED_LOCAL, 1, 0, 0)], [0], (1, 0, 1, 0))
    assert ex.value.code == _lib.EINVAL
    with pytest.raises(_lib.P3GpuError) as ex:
        gpu.air_program_create_layout(f.id, [(PERIODIC, 1, 0, 0)], [0], (1, 0, 0, 1))
    assert ex.value.code == _lib.EINVAL
    assert gpu.launches == n0


# ---------------------------------------------------------------- proofs: GPU bytes == stand-in device bytes, both verifiers accept
@pytest.mark.parametrize("name", list(ROUND_TRIPS))
def test_gpu_proof_equals_stand_in_proof(gpu, name, monkeypatch):
    import stark_verify as V
    import stark_verify_layout as VL
    from plonky3_b200.proof_io import proof_from_postcard
    from plonky3_b200.uni_stark import prove, setup_preprocessed, verify
    log_n, fri = ROUND_TRIPS[name]
    n = 1 << log_n
    config, cfg = _config(gpu, fri, device_challenger=True)
    air, trace = _air_and_trace(name, n, gpu)
    setup = setup_preprocessed(config, air, log_n)
    data, vk = setup if setup else (None, None)
    commits = []                                                        # pcs.commit calls: the trace's, one per proof
    commit = config.pcs.commit
    monkeypatch.setattr(config.pcs, "commit", lambda evals: commits.append(len(evals)) or commit(evals))
    raw = prove(config, air, dev(trace), preprocessed=data).to_postcard()
    verify(V.product_config(BabyBear, cfg), air, raw, preprocessed_vk=vk)
    sv_vk = None if vk is None else {"width": vk.width, "degree_bits": vk.degree_bits, "commitment": vk.commitment}
    VL.verify(V.Fld(BabyBear.id), cfg, X.stark_verify_air(name), proof_from_postcard(raw), preprocessed_vk=sv_vk)
    if data is not None:                                                # the prover data serves a second proof without a new commit
        assert prove(config, air, dev(trace), preprocessed=data).to_postcard() == raw
        assert commits == [1, 1]
    # the same driver on the oracle-backed stand-in device writes the same bytes
    mock = LayoutMockGpu()
    mconfig, _ = _config(mock, fri)
    mair, _ = _air_and_trace(name, n, mock)
    msetup = setup_preprocessed(mconfig, mair, log_n)
    with monkeypatch.context() as mp:
        mp.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
        mraw = prove(mconfig, mair, torch.from_numpy(trace.view(np.int32)), preprocessed=msetup[0] if msetup else None).to_postcard()
    assert mraw == raw
