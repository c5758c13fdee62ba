"""GPU: the persistent GEMM, the flash-attention rings and the norm kernels at the UNet's production sizes, where each
CTA (or warp, or thread) runs many units of work in sequence and carries state from one to the next: the TMA ring and
its mbarrier phases across tiles, the accumulator restart, the epilogue staging tile, the K / V ring after many wraps,
the LayerNorm row prefetch, the gn_apply batches.

Every case first asserts the regime it claims (work items per CTA, ring wraps, rows per warp, batches per thread) from
the device's SM count and a mirror of the host-side sizing, so that a change to tiling or grid sizing fails here
instead of quietly shrinking the case. Then three checks:
  1. every element (or every row of a sample that covers each position of several CTAs' work sequences and the last,
     partial tile) within an fp64 bound, as in test_kernel_contract_gpu.py;
  2. bit for bit equal to the same problem launched in slices small enough that each CTA gets one work item: a
     result must not depend on where in the schedule its work ran (fp64-atomic GroupNorm statistics: to 1e-12);
  3. two launches of the same descriptor give the same bits."""
from __future__ import annotations

import math

import pytest
import torch
import torch.nn.functional as F

from tango_b200 import lib as L
from tango_b200 import ops
from test_kernel_contract_gpu import (GEMM_GAMMA, U32, Out, act_ref, attn_ref, bf, fused_buffer,
                                      gemm_plan_family, geglu_reference, geglu_weights, pack_split, poisoned,
                                      poisoned_flat, rand, row_view, rowcol_err, skip_concat, skip_concat_groups)

pytestmark = pytest.mark.gpu

BM = 128          # GEMM M tile (gemm_tc.cu)
FA_BN = 64        # keys per attention tile (attention.cu)
LN_WARPS = 8      # LayerNorm warps per CTA; grid capped at 4 CTAs per SM (elementwise.cu)
GN_BATCH = 8      # rows per gn_apply_rows batch (elementwise.cu)
TAPS3 = [(t // 3 - 1, t % 3 - 1) for t in range(9)]   # (dh, dw) of the packed 3x3 taps, tap-major
SCALE = 0.125


def num_sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def same_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Bitwise equality (NaN and -0.0 compare by their bits)."""
    it = {2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return a.shape == b.shape and torch.equal(a.contiguous().view(it), b.contiguous().view(it))


def excess_dev(got, ref, bound) -> float:
    """`excess` evaluated on the device (the outputs here are too large to copy to the host per check)."""
    got = got.double()
    if not torch.isfinite(got).all():
        return math.inf
    return ((got - ref.double()).abs() / bound.double().clamp_min(1e-300)).max().item()


# ---------------------------------------------------------------------------------------------------- GEMM schedule
class GemmSchedule:
    """The work items of one tng_conv_gemm launch as the kernel walks them: the M tiling of plan_gemm, block_n and
    ksplit from tng_gemm_plan, grid = min(work, SMs), CTA c runs items c, c + grid, c + 2 grid, ..."""

    def __init__(self, W, H, NB, Ncols, block_n, ksplit, sms):
        if W >= BM or H == 1:
            bw, bh, bn = BM, 1, 1
        else:
            bw = W
            rem = BM // bw
            bh, bn = (rem, 1) if H >= rem else (H, rem // H)
        self.W, self.H, self.NB, self.Ncols = W, H, NB, Ncols
        self.bw, self.bh, self.bn, self.block_n, self.ksplit = bw, bh, bn, block_n, ksplit
        self.tiles_w, self.tiles_h, self.tiles_n = -(-W // bw), -(-H // bh), -(-NB // bn)
        self.m_tiles = self.tiles_w * self.tiles_h * self.tiles_n
        self.n_tiles = -(-Ncols // block_n)
        self.work = self.m_tiles * self.n_tiles * ksplit
        self.grid = min(self.work, sms)

    def item(self, tile):
        """(M tile index, first output row, valid rows, N tile) of work item `tile` (mirrors work_item + nvalid)."""
        t2 = tile // self.ksplit
        tm, tn = t2 // self.n_tiles, t2 % self.n_tiles
        tw, th, tb = tm % self.tiles_w, (tm // self.tiles_w) % self.tiles_h, tm // (self.tiles_w * self.tiles_h)
        w0, h0, n0 = tw * self.bw, th * self.bh, tb * self.bn
        if self.bh == 1 and self.bn == 1:
            nvalid = min(BM, self.W - w0)
        elif self.bn == 1:
            nvalid = min(self.bh, self.H - h0) * self.bw
        else:
            nvalid = min(self.bn, self.NB - n0) * self.bh * self.bw
        return tm, (n0 * self.H + h0) * self.W + w0, nvalid, tn

    def sequence(self, c):
        return list(range(c, self.work, self.grid))

    def items_per_cta(self):
        return self.work // self.grid, -(-self.work // self.grid)

    def epilogue(self, tile, fast=True):
        """'full', 'partial-m' or 'partial-n': the epilogue shape the kernel takes for this (non-GEGLU) item."""
        _, _, nvalid, tn = self.item(tile)
        if (tn + 1) * self.block_n > self.Ncols:
            return "partial-n"
        return "full" if (fast and self.ksplit == 1 and nvalid == BM) else "partial-m"

    def sample_ctas(self):
        g = self.grid
        return sorted({0, 1, g // 2, g - 1})

    def sample_rows(self, device="cpu", extra_ctas=()):
        """Output rows of every work item of the sampled CTAs, and of the last (possibly partial) M tile."""
        rows = set()
        items = [t for c in self.sample_ctas() + list(extra_ctas) for t in self.sequence(c)] + [self.work - 1]
        for t in items:
            _, r0, nvalid, _ = self.item(t)
            rows.update(range(r0, r0 + nvalid))
        return torch.tensor(sorted(rows), dtype=torch.long, device=device)


def gemm_plan(views, groups, weight, W, H, NB, **kw):
    """(block_n, ksplit) tng_gemm_plan picks for this descriptor (one launch under the profiler; outputs are scratch)."""
    fam = gemm_plan_family(views, groups, weight, W, H, NB, **kw)
    bn = int(fam[len("gemm_tc<"):].split(",")[0].rstrip(">"))
    return bn, 2 if "splitk" in fam else 1


def im2col_rows(x, rows, taps):
    """x fp64 [NB, H, W, C] (channels last); rows: flat output-pixel indices -> [len(rows), len(taps) * C], tap-major,
    zero outside the image (a stride-1 'same' convolution's operand)."""
    NB, H, W, C = x.shape
    n, h, w = rows // (H * W), (rows // W) % H, rows % W
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    return torch.cat([xp[n, h + dh + 1, w + dw + 1] for dh, dw in taps], dim=1)


def gemm_rows_reference(x, rows, taps, wk, *, HW, bias=None, rowvec=None, res=None, alpha=1.0):
    """fp64 alpha * (conv(x) + bias + rowvec[image] + res) at `rows`, and the same on |operands| (the per-element scale
    of the fp32 summation error). wk: [Ncols, taps * C] (the packed weight without padding)."""
    a = im2col_rows(x, rows, taps)
    w = wk.double()
    y, ab = a @ w.t(), a.abs() @ w.abs().t()
    img = rows // HW
    for t in (bias, None if rowvec is None else rowvec[img], None if res is None else res[rows]):
        if t is not None:
            y, ab = y + t.double(), ab + t.double().abs()
    return alpha * y, abs(alpha) * ab


def slice_views(views, linear, a, b):
    """The A views of rows [a, b) (linear: rows on the W axis) or images [a, b) (convolution)."""
    if linear:
        return [L.View(v.t, v.C, b - a, 1, 1, v.s_w, v.s_h, v.s_n, v.off + a * v.s_w) for v in views]
    return [L.View(v.t, v.C, v.W, v.H, b - a, v.s_w, v.s_h, v.s_n, v.off + a * v.s_n) for v in views]


class GemmCase:
    """One tng_conv_gemm descriptor that can be launched whole or over a range of units (rows of a linear, images of a
    convolution) with every operand and output pointer offset to match."""

    def __init__(self, views, groups, weight, W, H, NB, *, linear, bias=None, rowvec=None, res=None, alias=False,
                 alpha=1.0, act=L.ACT_NONE, block_n=0, stats_hw=0):
        self.views, self.groups, self.weight, self.W, self.H, self.NB = views, groups, weight, W, H, NB
        self.linear, self.bias, self.rowvec, self.res, self.alias = linear, bias, rowvec, res, alias
        self.alpha, self.act, self.block_n, self.stats_hw = alpha, act, block_n, stats_hw
        self.units = W if linear else NB
        self.unit_rows = 1 if linear else H * W

    def launch(self, of=None, ob=None, st=None, a=0, b=None):
        b = self.units if b is None else b
        r0, r1 = a * self.unit_rows, b * self.unit_rows
        kw = dict(bias=self.bias, alpha=self.alpha, act=self.act, block_n=self.block_n)
        if self.rowvec is not None:
            kw["rowvec"] = self.rowvec[a:b]
        if self.alias:
            kw["res"] = of.view[r0:r1]
        elif self.res is not None:
            kw["res"] = self.res[r0:r1]
        if of is not None:
            kw["out_f32"] = of.view[r0:r1]
        if ob is not None:
            kw["out_bf16"], kw["split_off"] = ob.view[r0:r1], ob.split_off
        if st is not None:
            kw["gn_stats"], kw["stats_hw"] = st[a:b], self.stats_hw
        W, NB = (b - a, 1) if self.linear else (self.W, b - a)
        L.conv_gemm(slice_views(self.views, self.linear, a, b), self.groups, self.weight, W, self.H, NB, **kw)

    def schedule(self, sms):
        kw = dict(bias=self.bias, alpha=self.alpha, act=self.act, block_n=self.block_n)
        return GemmSchedule(self.W, self.H, self.NB, self.weight.shape[0], *self.plan(self.units, **kw), sms)

    def plan(self, units, **kw):
        rows = units * self.unit_rows
        Ncols = self.weight.shape[0]
        dev = self.weight.device
        if self.alias:
            kw["res"] = torch.zeros(rows, Ncols, device=dev)
        elif self.res is not None:
            kw["res"] = self.res[:rows]
        if self.rowvec is not None:
            kw["rowvec"] = self.rowvec[:units]
        views = slice_views(self.views, self.linear, 0, units)
        W, NB = (units, 1) if self.linear else (self.W, units)
        outs = {}
        if self.want_f32:
            outs["out_f32"] = kw["res"] if self.alias else torch.empty(rows, Ncols, device=dev)
        if self.want_bf16:
            outs["out_bf16"] = torch.empty(rows, 2 * Ncols + 8 if self.split_off else Ncols, device=dev,
                                           dtype=torch.bfloat16)
            outs["split_off"] = self.split_off
        if self.stats_hw:
            outs["gn_stats"] = torch.zeros(NB, Ncols, 2, dtype=torch.float64, device=dev)
            outs["stats_hw"] = self.stats_hw
        return gemm_plan(views, self.groups, self.weight, W, self.H, NB, **kw, **outs)

    want_f32, want_bf16, split_off = True, False, 0

    def slices(self, sched, sms):
        """Unit ranges small enough that each CTA gets one work item, cut at M-tile boundaries (whole tiles of images
        for a convolution)."""
        per_tile_units = BM if self.linear else sched.bn          # units in one M tile (or its image count)
        tiles_per_unit = 1 if self.linear else sched.tiles_w * sched.tiles_h
        per = max(1, sms // (sched.n_tiles * sched.ksplit * tiles_per_unit)) * per_tile_units
        if sched.work <= sms:      # already one item per CTA: one M tile per launch
            per = per_tile_units
        return [(a, min(a + per, self.units)) for a in range(0, self.units, per)]


def check_sliced_and_repeat(case, sched, sms, outs, make_outs, *, stats=None):
    """The whole launch (already in `outs`) against the sliced launches and against a second whole launch."""
    sl = make_outs()
    for a, b in case.slices(sched, sms):
        case.launch(*sl, a=a, b=b)
    rep = make_outs()
    case.launch(*rep)
    torch.cuda.synchronize()
    for big, one, two in zip(outs, sl, rep):
        if big is None:
            continue
        if isinstance(big, Out):
            assert same_bits(big.buf, one.buf), "sliced launches differ from the whole launch"
            assert same_bits(big.buf, two.buf), "two launches of one descriptor differ"
        else:   # fp64 GroupNorm statistics: atomics in arbitrary order
            tol = 1e-12 * stats.abs()
            assert excess_dev(one, big, tol) <= 1.0 and excess_dev(two, big, tol) <= 1.0


def slice_plans_match(case, sched, sms):
    """Every slice keeps the whole launch's block_n and ksplit and gives each CTA at most one work item."""
    for units in {b - a for a, b in case.slices(sched, sms)}:
        s = case_schedule(case, units, sms)
        assert (s.block_n, s.ksplit) == (sched.block_n, sched.ksplit)
        assert s.work <= sms
    return len(case.slices(sched, sms))


def case_schedule(case, units, sms):
    kw = dict(bias=case.bias, alpha=case.alpha, act=case.act, block_n=case.block_n)
    W, NB = (units, 1) if case.linear else (case.W, units)
    return GemmSchedule(W, case.H, NB, case.weight.shape[0], *case.plan(units, **kw), sms)


def report_gemm(name, sched, e, n_slices):
    lo, hi = sched.items_per_cta()
    print(f"{name}: block_n={sched.block_n} ksplit={sched.ksplit} {sched.m_tiles} M x {sched.n_tiles} N tiles, "
          f"grid {sched.grid}, {lo}-{hi} work items per CTA, {n_slices} sliced launches; worst excess {e:.3f}")


# ---------------------------------------------------------------------------------------------------- GEMM cases
def linear_case(g, cuda, rows, Cin, Ncols, *, w=None, **kw):
    x = poisoned(bf(rand(g, rows, Cin)).to(cuda))
    wk = bf(rand(g, Ncols, Cin, scale=Cin ** -0.5) if w is None else w)
    wt = poisoned(wk.to(cuda), col_pad=8, row_pad=0)
    case = GemmCase([row_view(x, 1, 1, rows)], [(0, 0, 0, 0, 0, (Cin + 63) // 64)], wt, rows, 1, 1, linear=True, **kw)
    return case, x, wk


def test_gemm_out_projection_residual_aliases_output(cuda):
    """65536 x 320 x 320 with an fp32 residual that IS the output (the transformer out-projection: res == out_f32),
    bias and alpha: every chunk's loads are issued before its stores, on every work item of the sequence."""
    sms = num_sms()
    g = torch.Generator().manual_seed(1)
    rows, Cin, Ncols = 65536, 320, 320
    res0 = rand(g, rows, Ncols).to(cuda)
    case, x, wk = linear_case(g, cuda, rows, Cin, Ncols, bias=rand(g, Ncols).to(cuda), alias=True, alpha=0.75,
                              block_n=0)
    sched = case.schedule(sms)
    assert sched.items_per_cta()[0] >= 3
    case.block_n = sched.block_n          # the slices keep the whole launch's N tile
    n_sl = slice_plans_match(case, sched, sms)
    make = lambda: (Out(rows, Ncols, dtype=torch.float32, device=cuda, ld=Ncols + 8, init=res0), None, None)
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    rs = sched.sample_rows(cuda)
    y, ab = gemm_rows_reference(x.double().view(1, 1, rows, Cin), rs, [(0, 0)], wk.to(cuda), HW=rows,
                                bias=case.bias, res=res0, alpha=case.alpha)
    got = outs[0].hi[rs]
    e = excess_dev(got, y, GEMM_GAMMA * ab + U32 * y.abs())
    assert e <= 1.0 and rowcol_err(got, y) < 1e-3
    assert outs[0].sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make)
    report_gemm("out-projection 65536x320x320, res == out", sched, e, n_sl)


@pytest.mark.parametrize("split", [False, True])
def test_gemm_qkv_projection(cuda, split):
    """QKV 65536 x 960 (K 320), bf16 output or hi/lo with a gap before the lo half."""
    sms = num_sms()
    g = torch.Generator().manual_seed(2 + split)
    rows, Cin, Ncols = 65536, 320, 960
    case, x, wk = linear_case(g, cuda, rows, Cin, Ncols)
    case.want_f32, case.want_bf16, case.split_off = False, True, (Ncols + 8 if split else 0)
    sched = case.schedule(sms)
    assert sched.items_per_cta()[0] >= 3
    case.block_n = sched.block_n
    n_sl = slice_plans_match(case, sched, sms)
    make = lambda: (None, Out(rows, Ncols, dtype=torch.bfloat16, device=cuda, split_off=case.split_off), None)
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    rs = sched.sample_rows(cuda)
    y, ab = gemm_rows_reference(x.double().view(1, 1, rows, Cin), rs, [(0, 0)], wk.to(cuda), HW=rows)
    ob = outs[1]
    sb = GEMM_GAMMA * ab
    e = excess_dev(ob.hi[rs], y, sb + 2.0 ** -8 * y.abs())
    if split:
        e = max(e, excess_dev(ob.value()[rs], y, sb + 2.0 ** -16 * y.abs()))
    assert e <= 1.0 and ob.sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make)
    report_gemm(f"QKV 65536x960 {'hi/lo' if split else 'bf16'}", sched, e, n_sl)


def test_gemm_geglu_feed_forward(cuda):
    """GEGLU 65536 x 2560 -> 1280 (K 320), block_n 256, erf form: ten N tiles per M tile, so every CTA's sequence
    walks through all of them."""
    sms = num_sms()
    g = torch.Generator().manual_seed(4)
    rows, Cin, Ncols, bn = 65536, 320, 2560, 256
    w, bias = geglu_weights(g, Ncols, bn, Cin)
    case, x, wk = linear_case(g, cuda, rows, Cin, Ncols, w=w, bias=bias.to(cuda), act=L.ACT_GEGLU, block_n=bn)
    case.want_f32, case.want_bf16 = False, True
    sched = case.schedule(sms)
    assert sched.block_n == bn and sched.items_per_cta()[0] >= 3
    tns = [{sched.item(t)[3] for t in sched.sequence(c)} for c in sched.sample_ctas()]
    assert min(map(len, tns)) >= 3 and set().union(*tns) == set(range(10))     # the sample sees every N tile
    n_sl = slice_plans_match(case, sched, sms)
    make = lambda: (None, Out(rows, Ncols // 2, dtype=torch.bfloat16, device=cuda), None)
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    rs = sched.sample_rows(cuda)
    y, ab = gemm_rows_reference(x.double().view(1, 1, rows, Cin), rs, [(0, 0)], wk.to(cuda), HW=rows, bias=case.bias)
    z, bound = geglu_reference(y, ab, bn, False)
    e = excess_dev(outs[1].hi[rs], z, bound + 2.0 ** -8 * z.abs())
    assert e <= 1.0 and outs[1].sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make)
    report_gemm("GEGLU 65536x2560->1280 erf", sched, e, n_sl)


def test_gemm_resnet_conv_skip_concat(cuda):
    """conv3x3 16 x 256 x 16 over a 320 + 320 skip concatenation (two NaN-padded views) -> 320 with bias, the per-image
    time-embedding vector, an fp32 residual, GroupNorm statistics fused in the epilogue, and fp32 + SiLU bf16 outputs."""
    sms = num_sms()
    g = torch.Generator().manual_seed(5)
    NB, H, W, chans, a0s, Cout = 16, 256, 16, (320, 320), (16, 8), 320
    rows, Cs = NB * H * W, sum(chans)
    views, data = skip_concat(g, cuda, NB, H, W, chans, a0s)
    groups, _ = skip_concat_groups(chans, a0s)
    wt = bf(rand(g, Cout, Cs, 3, 3, scale=(9 * Cs) ** -0.5))
    wk = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cs)
    w = poisoned(wk.to(cuda), col_pad=8, row_pad=0)
    res = poisoned(rand(g, rows, Cout).to(cuda))
    case = GemmCase(views, groups, w, W, H, NB, linear=False, bias=rand(g, Cout).to(cuda),
                    rowvec=rand(g, NB, Cout, scale=2.0).to(cuda), res=res, alpha=1.0, act=L.ACT_SILU,
                    stats_hw=H * W)
    case.want_bf16 = True
    sched = case.schedule(sms)
    assert sched.ksplit == 1 and sched.items_per_cta()[0] >= 3
    assert all(sched.epilogue(t) == "full" for t in range(sched.work))     # the fused-statistics epilogue
    case.block_n = sched.block_n
    n_sl = slice_plans_match(case, sched, sms)
    make = lambda: (Out(rows, Cout, dtype=torch.float32, device=cuda), Out(rows, Cout, dtype=torch.bfloat16,
                                                                            device=cuda),
                    torch.zeros(NB, Cout, 2, dtype=torch.float64, device=cuda))
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    of, ob, st = outs
    xc = torch.cat([d.double() for d in data], dim=1).view(NB, H, W, Cs)
    rs = sched.sample_rows(cuda)
    y, ab = gemm_rows_reference(xc, rs, TAPS3, wk.to(cuda), HW=H * W, bias=case.bias, rowvec=case.rowvec,
                                res=res.double())
    del xc
    sb = GEMM_GAMMA * ab
    e = excess_dev(of.hi[rs], y, sb + U32 * y.abs())
    z = act_ref(y, L.ACT_SILU)
    e = max(e, excess_dev(ob.hi[rs], z, 1.1 * sb + 2.0 ** -8 * z.abs()))
    # statistics = column sums of what was stored: fp32 partials over <= 128 rows, fp64 across partials
    o = of.hi.double().view(NB, H * W, Cout)
    sabs = o.abs().sum(1)
    e = max(e, excess_dev(st[..., 0], o.sum(1), 128 * U32 * sabs),
            excess_dev(st[..., 1], (o * o).sum(1), 128 * U32 * (o * o).sum(1)))
    assert e <= 1.0 and of.sentinel_intact() and ob.sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make, stats=torch.stack([sabs, (o * o).sum(1)], -1))
    report_gemm("conv3x3 16x256x16 (320+320)->320 + GN stats", sched, e, n_sl)


def test_gemm_ragged_rows_and_columns(cuda):
    """30000 rows (the last M tile has 48) x 584 columns at block_n 128 (five N tiles, the last 72 wide): a CTA's
    sequence runs the FULL epilogue, the predicated one for the partial N tile and the one for the partial M tile in
    turn, with bias, a bf16 residual and fp32 + SiLU hi/lo outputs."""
    sms = num_sms()
    g = torch.Generator().manual_seed(6)
    rows, Cin, Ncols = 30000, 192, 584
    case, x, wk = linear_case(g, cuda, rows, Cin, Ncols, bias=rand(g, Ncols).to(cuda), alpha=0.5, act=L.ACT_SILU,
                              res=poisoned(bf(rand(g, rows, Ncols)).to(cuda), col_pad=16), block_n=128)
    case.want_bf16, case.split_off = True, Ncols + 8
    sched = case.schedule(sms)
    assert sched.block_n == 128 and sched.items_per_cta()[0] >= 3
    mixed = [c for c in range(sched.grid) if {sched.epilogue(t) for t in sched.sequence(c)} ==
             {"full", "partial-n", "partial-m"}]
    assert mixed, "no CTA runs all three epilogue shapes"
    n_sl = slice_plans_match(case, sched, sms)
    make = lambda: (Out(rows, Ncols, dtype=torch.float32, device=cuda, ld=Ncols + 12),
                    Out(rows, Ncols, dtype=torch.bfloat16, device=cuda, split_off=case.split_off), None)
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    rs = sched.sample_rows(cuda, extra_ctas=mixed[:1])
    y, ab = gemm_rows_reference(x.double().view(1, 1, rows, Cin), rs, [(0, 0)], wk.to(cuda), HW=rows,
                                bias=case.bias, res=case.res.double(), alpha=case.alpha)
    of, ob = outs[0], outs[1]
    sb = GEMM_GAMMA * ab
    e = excess_dev(of.hi[rs], y, sb + U32 * y.abs())
    z = act_ref(y, L.ACT_SILU)
    e = max(e, excess_dev(ob.value()[rs], z, 1.1 * sb + 2.0 ** -16 * z.abs()),
            excess_dev(ob.hi[rs], z, 1.1 * sb + 2.0 ** -8 * z.abs()))
    assert e <= 1.0 and of.sentinel_intact() and ob.sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make)
    report_gemm(f"ragged 30000x584 (CTA {mixed[0]} runs full, partial-N and partial-M tiles)", sched, e, n_sl)


def test_gemm_underfilled_split_k_conv(cuda):
    """The 32 x 2 level (16 images, 1280 -> 1280 channels): 8 M tiles, so the plan splits K between two CTAs per output
    tile that red.add their partials; the result must not depend on which half lands first."""
    sms = num_sms()
    g = torch.Generator().manual_seed(7)
    NB, H, W, Cin, Cout = 16, 32, 2, 1280, 1280
    rows = NB * H * W
    x = poisoned(bf(rand(g, rows, Cin)).to(cuda))
    wt = rand(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    pc = ops.PackedConv(wt, rand(g, Cout), split=False, device=cuda)
    res = poisoned(rand(g, rows, Cout).to(cuda))
    case = GemmCase(ops.act_views(x, NB, H, W, Cin, False), pc.groups(), pc.weight, W, H, NB, linear=False,
                    bias=pc.bias, rowvec=rand(g, NB, Cout).to(cuda), res=res, alpha=0.5)
    sched = case.schedule(sms)
    assert sched.ksplit == 2 and sched.m_tiles == 8 and sched.items_per_cta()[1] <= 2
    # block_n stays automatic: split-K is only planned then (the slices plan the same N tile and split, checked below)
    n_sl = slice_plans_match(case, sched, sms)
    make = lambda: (Out(rows, Cout, dtype=torch.float32, device=cuda, ld=Cout + 4), None, None)
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    rs = torch.arange(rows, device=cuda)
    y, ab = gemm_rows_reference(x.double().view(NB, H, W, Cin), rs, TAPS3, bf(wt).permute(0, 2, 3, 1).reshape(
        Cout, 9 * Cin).to(cuda), HW=H * W, bias=pc.bias, rowvec=case.rowvec, res=res.double(), alpha=0.5)
    e = excess_dev(outs[0].hi, y, GEMM_GAMMA * ab + 2 * U32 * y.abs())    # one more rounding: the red.add
    assert e <= 1.0 and outs[0].sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make)
    report_gemm("split-K conv 16x32x2 1280->1280", sched, e, n_sl)


# ---------------------------------------------------------------------------------------------------- attention
def ring_wraps(Lk, nbuf):
    return -(-Lk // FA_BN) // nbuf


def attn_case_buffers(cuda, q, k, v, nsplit):
    """NaN-padded fused buffers (q alone, k | v side by side; hi | lo pairs in split mode) -> launch kwargs."""
    C = q.shape[1]
    if nsplit == 1:
        qbuf, (qc,) = fused_buffer([bf(q)], cuda)
        kvbuf, (kc, vc) = fused_buffer([bf(k), bf(v)], cuda)
        return dict(qbuf=qbuf, kvbuf=kvbuf, q_col0=qc, k_col0=kc, v_col0=vc), tuple(bf(t).to(cuda).double()
                                                                                      for t in (q, k, v))
    (qh, ql), (kh, kl), (vh, vl) = pack_split(q), pack_split(k), pack_split(v)
    qbuf, (qc, _) = fused_buffer([qh, ql], cuda, gap=0)
    kvbuf, (kc, _, vc, _) = fused_buffer([kh, kl, vh, vl], cuda, gap=0)
    lo = dict(q_lo_off=C, k_lo_off=C, v_lo_off=C)
    ref_ops = tuple(h.to(cuda).double() + l_.to(cuda).double() for h, l_ in ((qh, ql), (kh, kl), (vh, vl)))
    return dict(qbuf=qbuf, kvbuf=kvbuf, q_col0=qc, k_col0=kc, v_col0=vc, **lo), ref_ops


def attn_launch(bufs, out, *, B, heads, Lq, Lk, nsplit, kbias=None, sliced=False):
    """The whole launch, or one launch per (batch entry, head): q_col0 + 64 h, the batch entry's rows of every
    operand, its key-mask row and its output rows / columns."""
    b_ = dict(bufs)
    qbuf, kvbuf = b_.pop("qbuf"), b_.pop("kvbuf")
    if not sliced:
        L.attention(qbuf, kvbuf, kvbuf, out.view, batch=B, heads=heads, Lq=Lq, Lk=Lk, scale=SCALE, kbias=kbias,
                    nsplit=nsplit, split_off=out.split_off, **b_)
        return
    lo = {k_: b_[k_] for k_ in ("q_lo_off", "k_lo_off", "v_lo_off") if k_ in b_}
    for b in range(B):
        kv = kvbuf[b * Lk:(b + 1) * Lk]
        for h in range(heads):
            L.attention(qbuf[b * Lq:(b + 1) * Lq], kv, kv, out.view[b * Lq:(b + 1) * Lq, 64 * h:], batch=1, heads=1,
                        Lq=Lq, Lk=Lk, scale=SCALE, q_col0=b_["q_col0"] + 64 * h, k_col0=b_["k_col0"] + 64 * h,
                        v_col0=b_["v_col0"] + 64 * h, kbias=None if kbias is None else kbias[b * Lk:(b + 1) * Lk],
                        nsplit=nsplit, split_off=out.split_off, **lo)


def attn_excess(out, ref_ops, *, B, heads, Lq, Lk, nsplit, kbias=None):
    """Every output element against fp64 attention (one batch entry at a time: the score matrices of all of them do
    not fit the memory budget), with the bounds of test_kernel_contract_gpu.run_attention_case."""
    q, k, v = ref_ops
    C = heads * 64
    e = 0.0
    for b in range(B):
        rq, rk = slice(b * Lq, (b + 1) * Lq), slice(b * Lk, (b + 1) * Lk)
        ref, pv = attn_ref(q[rq], k[rk], v[rk], batch=1, heads=heads, Lq=Lq, Lk=Lk, scale=SCALE,
                           kbias=None if kbias is None else kbias[rk].view(1, Lk))
        if nsplit == 1:
            e = max(e, excess_dev(out.hi[rq], ref, 2.0 ** -7 * pv + 2.0 ** -8 * ref.abs()))
        else:
            e = max(e, excess_dev(out.value()[rq], ref, 2.0 ** -11 * pv + 2.0 ** -15 * ref.abs()))
    assert out.hi.shape[1] == C
    return e


def attn_three_checks(cuda, name, q, k, v, *, B, heads, Lq, Lk, nsplit, kbias=None, bufs=None):
    C = heads * 64
    bufs, ref_ops = attn_case_buffers(cuda, q, k, v, nsplit) if bufs is None else bufs
    kb = None if kbias is None else poisoned_flat(kbias.reshape(-1).to(cuda))
    so = C + 8 if nsplit == 2 else 0
    make = lambda: Out(B * Lq, C, dtype=torch.bfloat16, device=cuda, split_off=so, ld=(2 * C + 24) if so else C + 8)
    out = make()
    attn_launch(bufs, out, B=B, heads=heads, Lq=Lq, Lk=Lk, nsplit=nsplit, kbias=kb)
    torch.cuda.synchronize()
    assert out.sentinel_intact()
    e = attn_excess(out, ref_ops, B=B, heads=heads, Lq=Lq, Lk=Lk, nsplit=nsplit,
                    kbias=None if kbias is None else kbias.reshape(-1).to(cuda))
    sl, rep = make(), make()
    attn_launch(bufs, sl, B=B, heads=heads, Lq=Lq, Lk=Lk, nsplit=nsplit, kbias=kb, sliced=True)
    attn_launch(bufs, rep, B=B, heads=heads, Lq=Lq, Lk=Lk, nsplit=nsplit, kbias=kb)
    torch.cuda.synchronize()
    ctas = -(-Lq // 128) * heads * B
    print(f"{name}: {ctas} CTAs ({ctas / num_sms():.1f} per SM), {-(-Lk // FA_BN)} key tiles = "
          f"{ring_wraps(Lk, 3)} wraps of the 3-deep ring; worst excess {e:.3f}")
    assert e <= 1.0
    assert same_bits(out.buf, sl.buf), "per-(batch, head) launches differ from the whole launch"
    assert same_bits(out.buf, rep.buf), "two launches of one descriptor differ"
    return out, e


@pytest.fixture(scope="module")
def self_attn_operands():
    """q / k / v of the level-0 self-attention: B 16 x 5 heads x 4096 tokens (fp32, on the host)."""
    g = torch.Generator().manual_seed(11)
    B, heads, L_ = 16, 5, 4096
    return tuple(rand(g, B * L_, heads * 64, scale=0.7) for _ in range(3))


@pytest.mark.parametrize("grow", [False, True])
def test_attention_self_level0(cuda, self_attn_operands, grow):
    """B 16 x 5 heads x 4096 x 4096, bf16, no mask: every key tile is full and unmasked, so every tile takes the
    folded-scale softmax; 64 key tiles = 21 wraps of the 3-deep ring. `grow`: key magnitudes rise 0.5 -> 5 along the
    sequence, so the running maximum keeps moving long after the first tiles and every rescale matters."""
    B, heads, L_ = 16, 5, 4096
    q, k, v = self_attn_operands
    if grow:
        k = k * torch.linspace(0.5, 5.0, L_).repeat(B)[:, None]
    assert ring_wraps(L_, 3) >= 8 and L_ % FA_BN == 0
    attn_three_checks(cuda, f"self-attention 16x5x4096^2{' growing keys' if grow else ''}", q, k, v, B=B,
                      heads=heads, Lq=L_, Lk=L_, nsplit=1)


def test_attention_self_zero_kbias_takes_tail_path(cuda, self_attn_operands):
    """The same unmasked problem with an all-zero kbias: the masked (tail) softmax on every tile, with the scale as a
    separate rounding; held to the same per-element bound as the folded result."""
    B, heads, L_ = 16, 5, 4096
    q, k, v = self_attn_operands
    assert ring_wraps(L_, 3) >= 8
    attn_three_checks(cuda, "self-attention 16x5x4096^2, zero kbias", q, k, v, B=B, heads=heads, Lq=L_, Lk=L_,
                      nsplit=1, kbias=torch.zeros(B, L_))


def test_attention_split_mode(cuda):
    """The parity mode (hi/lo operands, three products per MMA) at B 2 x 5 heads x 4096: 1 CTA per SM, 21 ring wraps."""
    g = torch.Generator().manual_seed(12)
    B, heads, L_ = 2, 5, 4096
    q, k, v = (rand(g, B * L_, heads * 64, scale=0.7) for _ in range(3))
    assert ring_wraps(L_, 3) >= 8
    attn_three_checks(cuda, "split-mode self-attention 2x5x4096^2", q, k, v, B=B, heads=heads, Lq=L_, Lk=L_, nsplit=2)


def test_attention_cross_cfg_masks(cuda):
    """Cross-attention Lq 4096 x Lk 64 (text tokens), B 16 = 8 unconditional + 8 conditional rows with their own key
    masks (-10000 past each prompt's length): 2560 CTAs, the masked softmax on their one key tile."""
    g = torch.Generator().manual_seed(13)
    B, heads, Lq, Lk = 16, 5, 4096, 64
    C = heads * 64
    q = rand(g, B * Lq, C, scale=0.7)
    k, v = rand(g, B * Lk, C, scale=0.7), rand(g, B * Lk, C) + 0.5
    lens = [2] * 8 + [5, 9, 17, 33, 40, 63, 64, 1]
    kb = torch.zeros(B, Lk)
    for b, n in enumerate(lens):
        kb[b, n:] = -10000.0
    assert -(-Lq // 128) * heads * B >= 8 * num_sms()
    attn_three_checks(cuda, "cross-attention 16x5x4096x64, CFG masks", q, k, v, B=B, heads=heads, Lq=Lq, Lk=Lk,
                      nsplit=1, kbias=kb)


@pytest.mark.parametrize("B,L_", [(8, 4096), (1, 12288)])
def test_attention_wide_vae(cuda, B, L_):
    """tng_attention_wide (the VAE AttnBlock, one head of width 512; single K / V buffer refilled in line) at the 10 s
    (L 4096) and 30 s (L 12288) sizes: 64 / 192 key tiles per CTA. Key magnitudes grow along the sequence. Every
    output row of several query tiles (each covers all key tiles) against fp64; bit for bit per batch entry."""
    C = 512
    g = torch.Generator().manual_seed(14 + L_)
    q = bf(rand(g, B * L_, C))
    k = bf(rand(g, B * L_, C) * torch.linspace(1.0, 2.5, L_).repeat(B)[:, None])
    v = bf(rand(g, B * L_, C) + 0.5)
    assert ring_wraps(L_, 1) >= 8
    buf, (qc, kc, vc) = fused_buffer([q, k, v], cuda)
    make = lambda: Out(B * L_, C, dtype=torch.bfloat16, device=cuda, col0=8, ld=C + 24)

    def launch(out, b0=0, b1=B):
        rows = slice(b0 * L_, b1 * L_)
        L.attention_wide(buf[rows], buf[rows], buf[rows], out.view[rows], batch=b1 - b0, L=L_, dim=C, scale=C ** -0.5,
                         q_col0=qc, k_col0=kc, v_col0=vc)

    out = make()
    launch(out)
    torch.cuda.synchronize()
    assert out.sentinel_intact()
    nq = L_ // 128
    qtiles = sorted({0, 1, nq // 2, nq - 1})
    e = 0.0
    for b in range(B):
        kd, vd = k[b * L_:(b + 1) * L_].to(cuda).double(), v[b * L_:(b + 1) * L_].to(cuda).double()
        rows = torch.cat([torch.arange(t * 128, (t + 1) * 128) for t in qtiles]) + b * L_
        qd = q[rows].to(cuda).double()
        p = (qd @ kd.t() * C ** -0.5).softmax(-1)
        ref, pv = p @ vd, p @ vd.abs()
        e = max(e, excess_dev(out.hi[rows.to(cuda)], ref, 2.0 ** -7 * pv + 2.0 ** -8 * ref.abs()))
    sl, rep = make(), make()
    for b in range(B):
        launch(sl, b, b + 1)
    launch(rep)
    torch.cuda.synchronize()
    print(f"VAE attention B {B} x L {L_}: {2 * nq * B} CTAs, {ring_wraps(L_, 1)} key tiles through the single buffer; "
          f"worst excess {e:.3f} over query tiles {qtiles}")
    assert e <= 1.0
    assert same_bits(out.buf, sl.buf) and same_bits(out.buf, rep.buf)


# ---------------------------------------------------------------------------------------------------- LayerNorm / RMSNorm
def ln_rows_per_warp(rows, sms):
    warps = min(-(-rows // LN_WARPS), 4 * sms) * LN_WARPS
    return rows / warps, warps


def ln_operands(g, cuda, rows, Cc):
    """Rows with their own offsets (-50 .. 50) and scales (0.5 .. 2), so a row normalised with another row's
    statistics is wrong by far more than the bound."""
    off = torch.linspace(-50.0, 50.0, rows)[torch.randperm(rows, generator=g)]
    sc = torch.linspace(0.5, 2.0, rows)[torch.randperm(rows, generator=g)]
    return (rand(g, rows, Cc) * sc[:, None] + off[:, None]).to(cuda)


@pytest.mark.parametrize("rms", [False, True])
def test_layernorm_rmsnorm_65536_rows(cuda, rms):
    """LayerNorm / RMSNorm over 65536 rows of 320: the grid is capped at 4 CTAs of 8 warps per SM, so every warp walks
    ~16 rows, normalising one while it prefetches the next. Bounds as in test_layernorm_rmsnorm_template_boundaries."""
    sms = num_sms()
    g = torch.Generator().manual_seed(20 + rms)
    rows, Cc = 65536, 320
    per_warp, warps = ln_rows_per_warp(rows, sms)
    assert rows > 4 * sms * LN_WARPS and per_warp >= 8
    x = ln_operands(g, cuda, rows, Cc)
    gamma, beta = rand(g, Cc).to(cuda), rand(g, Cc).to(cuda)
    ni = (Cc // 4 + 31) // 32
    xd = x.double()

    def make():
        y = Out(rows, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 4, ld=2 * Cc + 12)
        return y, (Out(rows, Cc, dtype=torch.float32, device=cuda, ld=Cc, row_pad=4) if rms else None)

    def launch(outs, r0=0, r1=rows):
        y, yf = outs
        if rms:
            L.rmsnorm(x[r0:r1], gamma, 1e-6, y.view[r0:r1], split_off=y.split_off, y_f32=yf.buf[r0:r1])
        else:
            L.layernorm(x[r0:r1], gamma, beta, 1e-5, y.view[r0:r1], split_off=y.split_off)

    outs = make()
    launch(outs)
    torch.cuda.synchronize()
    y, yf = outs
    if rms:
        ref = gamma.double() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6)
        rel = (2 * ni + 10) * U32
        e = max(excess_dev(y.value(), ref, (rel + 2.0 ** -16) * ref.abs() + 1e-30),
                excess_dev(yf.hi, ref, rel * ref.abs() + 1e-30))
    else:
        ref = F.layer_norm(xd, (Cc,), gamma.double(), beta.double(), 1e-5)
        rstd = 1.0 / (xd.var(-1, unbiased=False, keepdim=True) + 1e-5).sqrt()
        dmean = (2 * ni + 6) * U32 * xd.abs().mean(-1, keepdim=True)
        bound = dmean * rstd * gamma.double().abs() + 2.0 ** -16 * ref.abs() + 2.0 ** -18 * (beta.double().abs() + 1)
        e = excess_dev(y.value(), ref, bound)
    assert y.sentinel_intact() and (yf is None or yf.sentinel_intact())
    sl, rep = make(), make()
    step = 4 * sms * LN_WARPS               # one row per warp
    for r0 in range(0, rows, step):
        launch(sl, r0, min(r0 + step, rows))
    launch(rep)
    torch.cuda.synchronize()
    print(f"{'RMSNorm' if rms else 'LayerNorm'} 65536x320: {warps} warps, {per_warp:.1f} rows per warp, "
          f"{-(-rows // step)} sliced launches; worst excess {e:.3f}")
    assert e <= 1.0
    for a, b, r in zip(outs, sl, rep):
        if a is not None:
            assert same_bits(a.buf, b.buf), "sliced launches differ from the whole launch"
            assert same_bits(a.buf, r.buf), "two launches differ"


# ---------------------------------------------------------------------------------------------------- GroupNorm
def gn_slab(C, groups):
    """Channel slab per gn_apply CTA and the slab count (mirrors tng_groupnorm_apply)."""
    cpg = C // groups
    gps = 1
    while (gps * cpg) % 4 != 0 and gps < groups:
        gps += 1
    while gps * 2 * cpg <= 320 and groups % (gps * 2) == 0:
        gps *= 2
    if (gps * cpg) % 4 != 0 or groups % gps != 0:
        gps = groups
    return gps * cpg, groups // gps


def gn_apply_batches(NB, HW, C, groups, per_sm, sms):
    """(batches, batch size, last batch) of every thread of one image's gn_apply CTAs when `per_sm` CTAs are resident
    per SM (launch_gn_apply sizes the grid to one wave of them; gn_apply_rows splits a thread's rows into balanced
    batches of at most 8)."""
    slab, nslabs = gn_slab(C, groups)
    gx = max(1, per_sm * sms // (NB * nslabs))
    gn_rows = min(HW, max(8, -(-HW // gx)))
    QT = min(slab // 4, 256)
    RL = 256 // QT
    out = []
    for r0 in range(0, HW, gn_rows):
        nrows = min(gn_rows, HW - r0)
        for rl in range(RL):
            n = (nrows - rl + RL - 1) // RL
            if n <= 0:
                continue
            nb = -(-n // GN_BATCH)
            per = -(-n // nb)
            out.append((nb, per, n - (nb - 1) * per))
    return out


# 256-thread gn_apply CTAs resident per SM: its instantiations hold 74-80 registers per thread (sm_90a, CUDA 12.9), so
# the register file keeps at most 3 (launch_gn_apply asks the occupancy API); the premises hold for 1 to 4
GN_OCCUPANCY = range(1, 5)


@pytest.mark.parametrize("C0,C1,HW,groups", [(640, 320, 4096, 32), (320, 0, 4096, 32), (1280, 1280, 64, 32)])
def test_groupnorm_stats_and_apply(cuda, C0, C1, HW, groups):
    """groupnorm_stats + groupnorm_apply (SiLU, hi/lo output and a hi/lo raw copy) at NB 16: HW 4096 on a 640 + 320
    concatenation (fp32 + bf16 sources) and on 320 channels, where every thread of gn_apply runs several 8-row batches
    at any occupancy (on 320 channels some thread's last batch is ragged); and HW 64 on 2560 channels (eight slabs)."""
    sms = num_sms()
    NB = 16
    Cc = C0 + C1
    rows = NB * HW
    slab, nslabs = gn_slab(Cc, groups)
    if HW == 4096:
        for per_sm in GN_OCCUPANCY:
            bt = gn_apply_batches(NB, HW, Cc, groups, per_sm, sms)
            assert min(nb for nb, _, _ in bt) > 1, per_sm
            if C1 == 0:
                assert any(last < per for _, per, last in bt), per_sm
    else:
        assert nslabs >= 4
    g = torch.Generator().manual_seed(Cc + HW)
    x0 = (rand(g, rows, C0) * 2 + 0.5).to(cuda)
    x1 = bf(rand(g, rows, C1) - 0.3).to(cuda) if C1 else None
    gamma, beta = rand(g, Cc).to(cuda), rand(g, Cc).to(cuda)
    xs = [t for t in (x0, x1) if t is not None]

    def stats(a=0, b=NB):
        st = [torch.zeros(b - a, t.shape[1], 2, dtype=torch.float64, device=cuda) for t in xs]
        for t, s in zip(xs, st):
            L.groupnorm_stats(t[a * HW:b * HW], b - a, HW, s)
        return st

    def make():
        return (Out(rows, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 8, ld=2 * Cc + 24),
                Out(rows, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 16, ld=2 * Cc + 32))

    def apply(st, outs, a=0, b=NB):
        y, raw = outs
        r = slice(a * HW, b * HW)
        L.groupnorm(x0[r], st[0][a:b], None if x1 is None else x1[r], None if x1 is None else st[1][a:b], b - a, HW,
                    groups,
                    gamma, beta, 1e-5, L.ACT_SILU, y.view[r], split_off=y.split_off, raw=raw.view[r],
                    raw_split_off=raw.split_off)

    st = stats()
    outs = make()
    apply(st, outs)
    torch.cuda.synchronize()
    e = 0.0
    for t, s in zip(xs, st):
        xd = t.double().view(NB, HW, -1)
        e = max(e, excess_dev(s[..., 0], xd.sum(1), 128 * U32 * xd.abs().sum(1)),
                excess_dev(s[..., 1], (xd * xd).sum(1), 128 * U32 * (xd * xd).sum(1)))
    xc = torch.cat([t.double() for t in xs], dim=1)
    ref = F.silu(F.group_norm(xc.view(NB, HW, Cc).permute(0, 2, 1), groups, gamma.double(), beta.double(), 1e-5))
    ref = ref.permute(0, 2, 1).reshape(rows, Cc)
    y, raw = outs
    rms = ref.pow(2).mean().sqrt()
    e = max(e, excess_dev(y.value(), ref, 2.0 ** -16 * ref.abs() + 2.0 ** -18 * rms),
            excess_dev(y.hi, ref, 2.0 ** -8 * ref.abs() + 2.0 ** -18 * rms),
            excess_dev(raw.value(), xc, 2.0 ** -16 * xc.abs() + 1e-30))
    del ref
    assert y.sentinel_intact() and raw.sentinel_intact()
    # one image per launch (statistics and apply: the apply bit for bit), and a second whole launch
    st_sl = [torch.cat(parts) for parts in zip(*[stats(n, n + 1) for n in range(NB)])]
    sl, rep = make(), make()
    for n in range(NB):
        apply(st, sl, n, n + 1)
    st_rep = stats()
    apply(st, rep)
    torch.cuda.synchronize()
    for t, s, s2, s3 in zip(xs, st, st_sl, st_rep):
        xd = t.double().view(NB, HW, -1)
        mag = torch.stack([xd.abs().sum(1), (xd * xd).sum(1)], -1)
        # a repeat sums the same fp32 partials in another order; one image per launch sizes the partials differently
        # (gn_rows_for depends on NB), so there both are only within the fp32 bound of the exact sums
        assert excess_dev(s3, s, 1e-12 * mag) <= 1.0
        assert excess_dev(s2, s, 2 * 128 * U32 * mag) <= 1.0
    bt = {p: gn_apply_batches(NB, HW, Cc, groups, p, sms) for p in (2, 3, 4)}
    print(f"groupnorm NB 16 HW {HW} C {C0}+{C1}: {nslabs} slab(s) of {slab}; batches per thread at 2 / 3 / 4 CTAs "
          f"per SM: " + " / ".join(f"{min(b[0] for b in v)}-{max(b[0] for b in v)}" for v in bt.values()) +
          f"; worst excess {e:.3f}")
    assert e <= 1.0
    for a, b, r in zip(outs, sl, rep):
        assert same_bits(a.buf, b.buf), "per-image launches differ from the whole launch"
        assert same_bits(a.buf, r.buf), "two launches differ"
