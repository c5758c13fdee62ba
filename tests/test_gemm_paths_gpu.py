"""GPU: every epilogue cell of the persistent GEMM (tests/gemm_paths.py: the N x M tile instantiation, the epilogue body
and the run-time feature inside it) against fp64, through the launch audit of tests/launch_audit.py: the per-element
gemm_gamma(k) bound, a NaN-poisoned output region, every byte outside it unchanged, the GroupNorm statistics.

CASES holds one deterministic launch per few cells; together they reach every cell of REACHABLE at 132 SMs (H100 SXM),
which test_gemm_paths_cpu.py checks without a GPU. Before each launch the statement's plan must equal tng_gemm_plan at
the device's SM count, and the launch must still reach every cell it reaches at 132 SMs. Each case is launched twice into
fresh buffers over identical inputs: the outputs must agree bit for bit (split-K included), the fused statistics up to
the order of their fp64 additions. A seeded sweep of random descriptors adds the feature interactions no case names."""
from __future__ import annotations

import random
import time
from collections import Counter, defaultdict
from dataclasses import dataclass

import pytest
import torch

import gemm_paths as P
from launch_audit import install_audit
from tango_b200 import lib as L
from test_kernel_contract_gpu import (Out, bf, poisoned, poisoned_flat, rand, row_view, skip_concat,
                                      skip_concat_groups)

pytestmark = pytest.mark.gpu

SXM_SMS = 132          # H100 SXM: the SM count the committed case list is planned for


# ---------------------------------------------------------------------------------------------------- one launch
@dataclass(frozen=True)
class Case:
    """One tng_conv_gemm launch. taps: 1 (1 x 1 over the grid), 9 (3 x 3, padding 1) or a tuple of channel counts (a
    3 x 3 skip concatenation, one view per source with a_c0 > 0 and an element offset). res: None, torch.float32,
    torch.bfloat16 or "alias" (the fp32 output itself). mis: the one operand placed off its 16-byte alignment
    ("bias", "rowvec", "res", "f32", "bf16"), or "" ."""
    name: str
    W: int
    H: int
    NB: int
    Cin: int
    Ncols: int
    block_n: int = 0
    taps: object = 1
    bias: bool = True
    rowvec: bool = False
    res: object = None
    f32: bool = True
    bf16: bool = False
    split: bool = False
    act: int = L.ACT_NONE
    alpha: float = 1.0
    accumulate: bool = False
    stats_hw: int = 0
    mis: str = ""
    seed: int = 0

    @property
    def rows(self):
        return self.NB * self.H * self.W

    def build(self, dev, data=True):
        """(launch arguments of lib.conv_gemm, (fp32 Out, bf16 Out, statistics)) on dev; without data the operands
        hold zeros (the descriptor is all the CPU statement needs)."""
        g = torch.Generator().manual_seed(self.seed)
        mk = (lambda *s, scale=1.0: rand(g, *s, scale=scale)) if data else (lambda *s, scale=1.0: torch.zeros(*s))
        rows, N, mis = self.rows, self.Ncols, self.mis
        if isinstance(self.taps, tuple):
            a0s = tuple(8 * (i + 1) for i in range(len(self.taps)))
            views, _ = skip_concat(g, dev, self.NB, self.H, self.W, self.taps, a0s)
            groups, K = skip_concat_groups(self.taps, a0s)
        else:
            x = poisoned(bf(mk(rows, self.Cin)).to(dev))
            views, nkb = [row_view(x, self.NB, self.H, self.W)], (self.Cin + 63) // 64
            taps = [(0, 0)] if self.taps == 1 else [(t % 3 - 1, t // 3 - 1) for t in range(9)]
            groups, K = [(0, 0, dw, dh, t * self.Cin, nkb) for t, (dw, dh) in enumerate(taps)], len(taps) * self.Cin
        weight = poisoned(bf(mk(N, K, scale=K ** -0.5)).to(dev), col_pad=8, row_pad=0)
        kw = dict(alpha=self.alpha, accumulate=self.accumulate, act=self.act, act_param=0.2, block_n=self.block_n)
        if self.bias:
            kw["bias"] = poisoned_flat(mk(N).to(dev), lead=1 if mis == "bias" else 4)
        if self.rowvec:
            ld = N + 4 if N % 4 == 0 else N + 3
            rv = poisoned_flat(mk(self.NB * ld, scale=2.0).to(dev), lead=1 if mis == "rowvec" else 4)
            kw.update(rowvec=rv, rowvec_ld=ld)
        geglu = self.act in P.GEGLU_ACTS
        width = N // 2 if geglu else N
        prior = mk(rows, N).to(dev) if self.accumulate or self.res == "alias" else None
        of = Out(rows, N, dtype=torch.float32, device=dev, col0=1 if mis == "f32" else 0, init=prior) \
            if self.f32 else None
        ob = None
        if self.bf16:
            c0 = 2 if mis == "bf16" else 0
            so = (width + 15) // 8 * 8 if self.split else 0
            ob = Out(rows, width, dtype=torch.bfloat16, device=dev, col0=c0, split_off=so,
                     ld=(c0 + so + width + 15) // 8 * 8)
        if self.res == "alias":
            kw["res"] = of.view
        elif self.res is not None:
            kw["res"] = poisoned(mk(rows, N).to(self.res).to(dev), col0=3 if mis == "res" else 0)
        st = None
        if self.stats_hw:
            st = torch.zeros(rows // self.stats_hw, N, 2, dtype=torch.float64, device=dev)
            kw.update(gn_stats=st, stats_hw=self.stats_hw)
        kw.update(out_f32=None if of is None else of.view, out_bf16=None if ob is None else ob.view,
                  split_off=0 if ob is None else ob.split_off)
        return (views, groups, weight, self.W, self.H, self.NB), kw, (of, ob, st)

    def desc(self, dev="cpu"):
        args, kw, _ = self.build(dev, data=False)
        return P.desc_of(*args, **kw)


# ---------------------------------------------------------------------------------------------------- the case list
def _mode_case(bn, bm, mode, kind, seed):
    """Case of kind A (full tiles, per-warp row vector, fused statistics, SiLU + hi/lo where the statistics allow),
    B (ragged: full and partial tiles, more work items than SMs, per-slot row vector, accumulate, LReLU; statistics by
    the after-pass at 128 rows), C (misaligned: the SCALAR body), D (full tiles, the other activation of modes 4/5),
    E (ragged W-tiled rows, per-warp row vector, plain bf16 output, after-pass statistics) or F (256 rows: full tiles of
    eight 8-pixel images, after-pass statistics), for output mode `mode` on BN x BM tiles."""
    res = (torch.bfloat16 if (bn + mode) % 3 == 0 else torch.float32) if mode & 1 else None
    f32, bf16 = bool(mode & 2), bool(mode & 4)
    base = dict(res=res, f32=f32, bf16=bf16, seed=seed, block_n=bn if bm == 128 else 0)
    name = f"{kind} {bn}x{bm} mode {mode}"
    if bm == 128:
        N = 2 * bn
        if kind == "A":
            taps = 9 if mode in (3, 6) else 1
            grid = dict(W=16, H=16, NB=2) if taps == 9 else dict(W=512, H=1, NB=1)
            return Case(name, **grid, Cin=72, Ncols=N, taps=taps, rowvec=True, stats_hw=256,
                        act=L.ACT_SILU if mode & 6 == 6 else L.ACT_NONE, split=mode & 6 == 6, **base)
        if kind == "B":
            act = {4: L.ACT_SILU, 5: L.ACT_LRELU}.get(mode, L.ACT_LRELU if bf16 else L.ACT_NONE)
            return Case(name, W=4, H=2, NB=16 * 66 + 5, Cin=64, Ncols=N, rowvec=True, accumulate=f32, act=act,
                        split=mode in (4, 5), stats_hw=0 if mode in (4, 5) else 8, alpha=0.75, **base)
        if kind == "C":
            mis = {2: "bias", 3: "res", 4: "bias", 5: "bf16", 6: "rowvec", 7: "f32"}[mode]
            slot = dict(W=2, H=2, NB=50)          # 4 rows per image: the per-slot row vector
            feats = {2: dict(accumulate=True, stats_hw=100), 3: dict(accumulate=True, rowvec=True),
                     4: dict(**slot, rowvec=True, stats_hw=4), 5: dict(**slot, rowvec=True, act=L.ACT_SILU, split=True),
                     6: dict(act=L.ACT_LRELU, accumulate=True, rowvec=True, stats_hw=100),
                     7: dict(act=L.ACT_SILU, split=True, accumulate=True, rowvec=True)}[mode]
            feats = {"W": 200, "H": 1, "NB": 1, **feats}
            return Case(name, Cin=72, Ncols=N - 4, mis=mis, alpha=0.5, **{**base, **feats})
        if kind == "D":
            return Case(name, W=256, H=1, NB=1, Cin=136, Ncols=N, act=L.ACT_LRELU if mode == 4 else L.ACT_SILU,
                        **base)
        if kind == "E":
            return Case(name, W=300, H=1, NB=1, Cin=72, Ncols=N, rowvec=True, stats_hw=100, **base)
    else:   # 256-row tiles: block_n 160 from the automatic choice, >= 64 K blocks, >= half a wave of work items
        if kind == "A":
            return Case(name, W=66 * 256, H=1, NB=1, Cin=4096, Ncols=160, rowvec=True, stats_hw=66 * 64,
                        act=L.ACT_SILU if mode & 6 == 6 else L.ACT_NONE, split=mode & 6 == 6, **base)
        if kind == "B":
            act = {4: L.ACT_SILU, 5: L.ACT_LRELU}.get(mode, L.ACT_LRELU if bf16 else L.ACT_NONE)
            return Case(name, W=4, H=2, NB=32 * 66 + 5, Cin=4096, Ncols=320, rowvec=True, accumulate=f32, act=act,
                        split=mode in (4, 5), alpha=0.75, **base)
        if kind == "D":
            return Case(name, W=66 * 256 + 100, H=1, NB=1, Cin=4096, Ncols=320, rowvec=True,
                        act=L.ACT_LRELU if mode == 4 else L.ACT_SILU, **base)
        if kind == "F":
            return Case(name, W=4, H=2, NB=32 * 66, Cin=4096, Ncols=160, stats_hw=8, **base)
    raise ValueError((bn, bm, kind))


def _geglu_cases():
    out = []
    for bn in (128, 256):
        # full and partial tiles (erf), more work items than SMs; the hi/lo and tanh forms on ragged or full rows
        for body, act, split, rows in (("erf", L.ACT_GEGLU, False, 66 * 128 + 40), ("erf-hilo", L.ACT_GEGLU, True, 300),
                                       ("tanh", L.ACT_GEGLU_TANH, False, 300), ("tanh-hilo", L.ACT_GEGLU_TANH, True, 256)):
            out.append(Case(f"GEGLU {bn} {body}", W=rows, H=1, NB=1, Cin=72, Ncols=2 * bn, block_n=bn, f32=False,
                            bf16=True, split=split, act=act, seed=bn + rows))
    return out


def constructed_cases():
    cases = []
    for i, bn in enumerate(P.BNS):
        for mode in P.MODES:
            for kind in "ABC" + ("DE" if mode in (4, 5) else ""):
                cases.append(_mode_case(bn, 128, mode, kind, seed=100 * i + 10 * mode + ord(kind)))
    for mode in P.MODES:
        for kind in "ABF" + ("D" if mode in (4, 5) else ""):
            cases.append(_mode_case(160, 256, mode, kind, seed=1000 + 10 * mode + ord(kind)))
    cases += _geglu_cases()
    # split-K on the automatic block_n 160 path (4 M tiles x 1-2 N tiles): 36 K blocks (even halves) over a 3 x 3
    # convolution with row vector, residual and after-pass statistics; 63 (odd: halves of 31 and 32) over a skip
    # concatenation of two views with a_c0 > 0, tap offsets and b_k0 > 0
    cases.append(Case("split-K even", W=16, H=16, NB=2, Cin=256, Ncols=320, taps=9, rowvec=True, res=torch.float32,
                      alpha=0.5, stats_hw=256, seed=7))
    cases.append(Case("split-K odd", W=16, H=16, NB=2, Cin=0, Ncols=160, taps=(72, 264), seed=8))
    return cases


CASES = constructed_cases()


# ---------------------------------------------------------------------------------------------------- checks
def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


RESULTS = {}        # case name -> (cells, worst excess)


def stats_partials_bound(of, ob, st_shape):
    """64 * 2^-53 of the sum of |partials| per statistic: fp32 sums of 16 rows of the stored output (the fused epilogue's
    partials; the after-pass adds longer ones, whose magnitudes sum to no more)."""
    o = (of.hi if of is not None else ob.hi).double()
    imgs, N = st_shape[0], st_shape[1]
    v = o.reshape(imgs, -1, 16, N) if (o.shape[0] // imgs) % 16 == 0 else o.reshape(imgs, -1, 1, N)
    s = v.sum(2).abs().sum(1)
    q = (v * v).sum(2).sum(1)
    return 64 * 2.0 ** -53 * torch.stack([s, q], -1)


def bits(t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int16)


def run_case(case, cuda, monkeypatch, sms, *, twice=True):
    """Plan parity, the launch under the audit, the cells it ran; twice: a second launch into fresh buffers."""
    launch = L.conv_gemm
    args, kw, outs = case.build(cuda)
    d = P.desc_of(*args, **kw)
    p = P.plan(d, sms)
    assert P.library_plan(d) == p.key, f"{case.name}: statement plan {p.key} != tng_gemm_plan {P.library_plan(d)}"
    got = P.cells(d, sms, p)
    audit = install_audit(monkeypatch, only=("conv_gemm",))
    n0 = L.launch_count()
    L.conv_gemm(*args, **kw)
    torch.cuda.synchronize()
    monkeypatch.undo()
    (rec,) = audit.records
    assert rec.family == p.family, (case.name, rec.family, p.family)
    assert L.launch_count() - n0 == rec.launches == (2 if p.stats == "after" else 1), (case.name, rec.launches, p.stats)
    if twice:
        args2, kw2, outs2 = case.build(cuda)
        launch(*args2, **kw2)
        torch.cuda.synchronize()
        for a, b in zip(outs[:2], outs2[:2]):
            if a is not None:
                assert torch.equal(bits(a.buf), bits(b.buf)), f"{case.name}: a second launch differs"
        if outs[2] is not None:
            bound = stats_partials_bound(outs[0], outs[1], outs[2].shape)
            assert ((outs[2] - outs2[2]).abs() <= bound).all(), f"{case.name}: statistics differ beyond their order"
    return got, p, rec.excess


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_gemm_cell(cuda, monkeypatch, case):
    sms = num_sms()
    want = P.cells(case.desc(cuda), SXM_SMS)
    got, p, e = run_case(case, cuda, monkeypatch, sms)
    lost = want - got
    assert not lost, f"{case.name} at {sms} SMs misses cells it reaches at {SXM_SMS}: {sorted(lost)}"
    RESULTS[case.name] = (got, e)
    print(f"{case.name}: {p.family} ksplit={p.ksplit} stats={p.stats} worst excess {e:.3f}")


def test_gemm_cell_matrix(cuda):
    """Prints the covered-cell matrix and the worst excess per body over the cases run in this session."""
    if not RESULTS:
        pytest.skip("no case of this module ran in this session")
    covered = set().union(*(c for c, _ in RESULTS.values()))
    worst = defaultdict(float)
    for cells, e in RESULTS.values():
        for bn, bm, body, _ in cells:
            worst[(bn, bm, body)] = max(worst[(bn, bm, body)], e)
    print(f"\n{len(covered & P.REACHABLE)} of {len(P.REACHABLE)} reachable cells covered by {len(RESULTS)} launches")
    print(P.matrix(covered))
    print("worst excess of a launch that ran the body:")
    for (bn, bm, body), e in sorted(worst.items()):
        print(f"  {bn:>3d} x {bm:<3d} {body:<18s} {e:.3f}")
    if len(RESULTS) == len(CASES):
        assert covered == P.REACHABLE, sorted(P.REACHABLE - covered)


# ---------------------------------------------------------------------------------------------------- random sweep
def random_case(rng: random.Random, i: int) -> Case:
    """A random valid-looking descriptor over the product of the features (small: <= ~2k rows, <= 640 K)."""
    geglu = rng.random() < 0.12
    shape = rng.choice(["linear", "images", "conv"])
    if shape == "linear":
        W, H, NB = rng.choice([64, 128, 200, 256, 384, 500, 640, 1000, 1536]), 1, 1
    else:
        W = rng.choice([1, 2, 4, 8, 16, 32, 64, 128])
        H = rng.choice([1, 2, 4, 8, 16, 32])
        NB = rng.randint(1, max(1, 2048 // (W * H)))
    taps = 9 if shape == "conv" else rng.choice([1, 1, (72, 136)]) if shape == "images" else 1
    Cin = rng.choice([8, 64, 72, 136, 200, 320, 640])
    if geglu:
        bn = rng.choice([128, 256])      # explicit: the audit's GEGLU reference needs the tile's hidden / gate split
        Ncols = rng.choice([256, 512]) if bn == 256 else rng.choice([128, 256, 384])
        return Case(f"sweep {i}", W, H, NB, Cin, Ncols, block_n=bn, taps=taps, bias=rng.random() < 0.8, f32=False,
                    bf16=True, split=rng.random() < 0.5, act=rng.choice(P.GEGLU_ACTS), seed=i)
    Ncols = rng.choice([4, 20, 32, 36, 64, 96, 128, 160, 192, 256, 320, 480, 512, 2, 6, 33, 100])
    f32 = rng.random() < 0.7
    bf16 = not f32 or rng.random() < 0.5
    res = rng.choice([None, None, torch.float32, torch.bfloat16] + (["alias"] if f32 else []))
    stats = rng.random() < 0.3
    return Case(f"sweep {i}", W, H, NB, Cin, Ncols, block_n=rng.choice([0, 0, 0, 32, 64, 128, 160, 256]), taps=taps,
                bias=rng.random() < 0.7, rowvec=rng.random() < 0.4, res=res, f32=f32, bf16=bf16,
                split=bf16 and rng.random() < 0.4, act=rng.choice([L.ACT_NONE, L.ACT_SILU, L.ACT_LRELU]),
                alpha=rng.choice([1.0, 0.5, -1.25]), accumulate=f32 and rng.random() < 0.3,
                stats_hw=(H * W if shape != "linear" else W // rng.choice([1, 2, 4])) if stats else 0,
                mis=rng.choice(["", "", "", "bias", "rowvec", "res", "f32", "bf16"]), seed=i)


def sweep_cases(n=200, seed=2024):
    """n random cases the planner accepts (drawn in order from one seeded stream)."""
    rng, out, i = random.Random(seed), [], 0
    while len(out) < n:
        c = random_case(rng, i)
        i += 1
        try:
            P.plan(c.desc(), 1)
        except P.Rejected:
            continue
        out.append(c)
    return out


def test_random_sweep(cuda, monkeypatch):
    sms = num_sms()
    hist, t0, worst = Counter(), time.time(), 0.0
    cases = sweep_cases()
    for c in cases:
        got, _, e = run_case(c, cuda, monkeypatch, sms, twice=False)
        hist.update(got)
        worst = max(worst, e)
    print(f"\nrandom sweep: {len(cases)} launches, {len(hist)} cells, worst excess {worst:.3f}, "
          f"{time.time() - t0:.1f} s")
    print(P.matrix(set(hist)))
    for (bn, bm, body, f), n in sorted(hist.items()):
        print(f"  {bn:>3d} x {bm:<3d} {body:<18s} {f:<12s} {n:4d}")
