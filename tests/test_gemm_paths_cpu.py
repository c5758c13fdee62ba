"""CPU: tests/gemm_paths.py states the GEMM planner (it agrees with tng_gemm_plan, which plans without a device, on
every sampled descriptor, acceptance and rejection included), its matrix of reachable cells is what the dispatch
reaches, and the constructed cases of test_gemm_paths_gpu.py cover that matrix at 132 SMs, each case needed."""
from __future__ import annotations

import random

import torch

import gemm_paths as P
from tango_b200 import lib as L
from test_gemm_paths_gpu import CASES, SXM_SMS, sweep_cases

BASE = 1 << 20          # fake, 256-byte aligned addresses: tng_gemm_plan reads none of them


def library_sms():
    """The SM count tng_gemm_plan plans for: the device's, or 1 without one (num_sms() in capi.cu)."""
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 1


def random_desc(rng: random.Random) -> P.Desc:
    """A descriptor over the whole feature space, invalid ones included (~1 in 3 is rejected)."""
    ch = rng.choice
    W = ch([1, 2, 3, 4, 8, 16, 24, 32, 64, 100, 128, 200, 256, 300, 512, 1000, 4096, 16896, 20000, 0])
    H = ch([1, 1, 2, 3, 4, 8, 16, 33, 64])
    NB = ch([1, 1, 2, 3, 5, 16, 64, 1000, 2117, -1])
    n_aviews = ch([1, 1, 1, 2, 3, 4, 0, 5])
    views = [(BASE + 4096 * i, ch([8, 64, 72, 320, 640, 4096, 12]), W, H, NB, 64, 64 * W, 64 * W * H)
             for i in range(max(n_aviews, 1))]
    n_groups = ch([1, 1, 2, 4, 9, 18, 40, 0, 41])
    Ktot = ch([64, 72, 320, 576, 2880, 4096, 11520])
    groups = []
    for _ in range(max(0, min(n_groups, 40))):
        view = ch([0] * 6 + list(range(n_aviews)) + [n_aviews])
        C = views[min(max(view, 0), len(views) - 1)][1]
        nkb = rng.randint(1, (C + 63) // 64) + ch([0] * 12 + [1])
        b_k0 = rng.randrange(0, Ktot, 8) + ch([0] * 12 + [Ktot])
        groups.append((view, ch([0, 0, 8, -8]), ch([-1, 0, 1]), ch([-1, 0, 1]), b_k0, nkb))
    Ncols = ch([1, 4, 20, 32, 36, 64, 96, 128, 160, 192, 256, 320, 480, 512, 640, 1280, 0])
    ptr = lambda p=0.5: BASE + 1024 * rng.randint(1, 64) + ch([0, 0, 0, 4, 8, 2]) if rng.random() < p else 0
    out_f32, out_bf16 = ptr(0.7), ptr(0.5)
    res = ch([0, ptr(1.0), out_f32])
    d = P.Desc(a=views[:max(n_aviews, 1)], g=groups, W=W, H=H, NB=NB, Ncols=Ncols, Ktot=Ktot,
               b=BASE, ldb=ch([0, 0, Ktot + 8, Ktot + 3]), bias=ptr(0.7), rowvec=ptr(0.3),
               rowvec_ld=ch([0, Ncols + 4, Ncols + 3]), res=res, res_dtype=ch([L.DT_F32, L.DT_BF16]),
               ldr=Ncols + ch([0, 4, 8, 3]), alpha=ch([1.0, 1.0, 0.5]), accumulate=int(rng.random() < 0.25),
               out_f32=out_f32, ld_f32=Ncols + ch([0, 4, 8, 1]), out_bf16=out_bf16, ld_bf16=Ncols + ch([0, 8, 16, 4]),
               act=ch([L.ACT_NONE, L.ACT_NONE, L.ACT_SILU, L.ACT_LRELU, L.ACT_GEGLU, L.ACT_GEGLU_TANH]),
               split_off=ch([0, 0, Ncols + 8, Ncols + 4]), block_n=ch([0, 0, 0, 0, 32, 64, 96, 128, 160, 256]),
               gn_stats=ptr(0.3), stats_hw=ch([W * H, 16, 8, W, 0, 7]), n_aviews=n_aviews, n_groups=n_groups)
    return d


def statement_plan(d, sms):
    try:
        return P.plan(d, sms).key
    except P.Rejected:
        return None


def test_statement_agrees_with_tng_gemm_plan():
    """Several hundred seeded random descriptors, the constructed cases and the random sweep of the GPU suite: the same
    accept / reject decision and, when accepted, the same block_n, M tile and ksplit."""
    sms = library_sms()
    rng = random.Random(1234)
    descs = [("random", random_desc(rng)) for _ in range(600)]
    descs += [(c.name, c.desc()) for c in CASES]
    descs += [(c.name, c.desc()) for c in sweep_cases(60)]
    accepted = 0
    for name, d in descs:
        want = P.library_plan(d)
        assert statement_plan(d, sms) == want, (name, d, want)
        accepted += want is not None
    assert 150 <= accepted <= len(descs) - 150, accepted     # both outcomes are well sampled


def test_statement_reaches_only_reachable_cells():
    """Every cell the statement's dispatch produces for the random descriptors and the GPU suite's random sweep, at 1,
    114 and 132 SMs, is in REACHABLE: an exclusion that is wrong fails here."""
    rng = random.Random(99)
    seen = set()
    descs = [random_desc(rng) for _ in range(600)] + [c.desc() for c in sweep_cases(300)]
    for d in descs:
        if d.W * d.H * d.NB > 1 << 16:
            continue
        for sms in (1, 114, SXM_SMS):
            try:
                seen |= P.cells(d, sms)
            except P.Rejected:
                break
    assert seen <= P.REACHABLE, sorted(seen - P.REACHABLE)
    assert len(seen) > 150


def test_reachable_matrix():
    assert len(P.REACHABLE) + len(P.EXCLUDED) == len(P.ALL_CELLS)
    assert all(isinstance(r, str) and r for r in P.EXCLUDED.values())
    insts = {(bn, bm) for bn, bm, _, _ in P.REACHABLE}
    assert insts == set(P.INSTANTIATIONS)
    bodies = {(bn, bm, body) for bn, bm, body, _ in P.REACHABLE}
    assert len(bodies) == 5 * 8 + 7 + 2 * 5      # the epilogue bodies gemm_tc_kernel compiles


def case_cells():
    return {c.name: P.cells(c.desc(), SXM_SMS) for c in CASES}


def test_constructed_cases_cover_reachable():
    cells = case_cells()
    covered = set().union(*cells.values())
    missing = P.REACHABLE - covered
    assert not missing, f"{len(missing)} reachable cells no constructed case reaches at {SXM_SMS} SMs: {sorted(missing)}"
    assert covered <= P.REACHABLE, sorted(covered - P.REACHABLE)


def test_every_constructed_case_is_needed():
    """Each case reaches a cell no other case reaches, so that deleting one fails the coverage test."""
    cells = case_cells()
    assert len(cells) == len(CASES), "two cases share a name"
    for name, own in cells.items():
        others = set().union(*(c for n, c in cells.items() if n != name))
        assert own - others, f"{name} reaches no cell of its own"


def test_after_pass_statistics_are_refused_before_the_gemm_runs():
    """gn_stats on a launch whose statistics come from the after-pass, with an output that pass cannot read (Ncols % 4,
    ld % 4, a 4-byte aligned fp32 output): tng_gemm_plan, and so tng_conv_gemm before it writes anything, returns
    TNG_EINVAL. Such a launch used to run the GEMM, then fail in the after-pass with the output written and the
    statistics not."""
    lib = L.load()
    base = dict(a=[(BASE, 64, 200, 1, 1, 64, 64 * 200, 64 * 200)], g=[(0, 0, 0, 0, 0, 1)], W=200, H=1, NB=1, Ktot=64,
                b=BASE, out_f32=BASE + 4096, gn_stats=BASE + 8192, stats_hw=100)
    good = P.Desc(Ncols=64, ld_f32=72, **base)
    assert P.library_plan(good) is not None and P.plan(good, 1).stats == "after"
    for bad in (dict(Ncols=62, ld_f32=72), dict(Ncols=64, ld_f32=70), dict(Ncols=64, ld_f32=72, out_f32=BASE + 4100)):
        d = P.Desc(**{**base, **bad})
        assert P.library_plan(d) is None, bad
        assert b"gn_stats" in lib.tng_last_error()
    ok8 = P.Desc(**{**base, "Ncols": 64, "ld_f32": 72, "out_f32": BASE + 4104})   # 8-byte aligned: the scalar epilogue
    assert P.library_plan(ok8) is not None and not P.plan(ok8, 1).fast_epi
