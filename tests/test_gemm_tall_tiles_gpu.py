"""GPU: the persistent GEMM on 256-row M tiles (block_n 160, long reductions). tng_gemm_plan reports the M tile; the
schedule below models the 256-row tiling (the same box rule as 128 rows: bw x bh x bn output pixels with product 256),
and every case runs the checks of test_kernels_at_scale_gpu.py: sampled rows of every work item against fp64, bit for
bit against launches of slices small enough to plan 128-row tiles (wgmma accumulates an output element in the same K
order wherever its row lies in the tile), and a repeat launch."""
from __future__ import annotations

import pytest
import torch

from tango_b200 import lib as L
from test_kernel_contract_gpu import (GEMM_GAMMA, U32, Out, act_ref, bf, gemm_plan_family, poisoned, rand, row_view,
                                      skip_concat, skip_concat_groups)
from test_kernels_at_scale_gpu import (TAPS3, GemmCase, GemmSchedule, check_sliced_and_repeat, excess_dev,
                                       gemm_rows_reference, num_sms, slice_views)

pytestmark = pytest.mark.gpu

SLICE_ROWS = 8192   # 32 M tiles of 256 rows x 2 N tiles: too few work items for 256 rows, <= 132 items at 128 rows


class TallSchedule(GemmSchedule):
    """GemmSchedule with an M tile of bm rows."""

    def __init__(self, W, H, NB, Ncols, block_n, bm, sms):
        super().__init__(W, H, NB, Ncols, block_n, 1, sms)
        if W >= bm or H == 1:
            bw, bh, bn = bm, 1, 1
        else:
            bw = W
            rem = bm // bw
            bh, bn = (rem, 1) if H >= rem else (H, rem // H)
        self.bm, self.bw, self.bh, self.bn = bm, bw, bh, bn
        self.tiles_w, self.tiles_h, self.tiles_n = -(-W // bw), -(-H // bh), -(-NB // bn)
        self.m_tiles = self.tiles_w * self.tiles_h * self.tiles_n
        self.work = self.m_tiles * self.n_tiles
        self.grid = min(self.work, sms)

    def item(self, tile):
        tm, tn = tile // self.n_tiles, tile % self.n_tiles
        tw, th, tb = tm % self.tiles_w, (tm // self.tiles_w) % self.tiles_h, tm // (self.tiles_w * self.tiles_h)
        w0, h0, n0 = tw * self.bw, th * self.bh, tb * self.bn
        if self.bh == 1 and self.bn == 1:
            nvalid = min(self.bm, self.W - w0)
        elif self.bn == 1:
            nvalid = min(self.bh, self.H - h0) * self.bw
        else:
            nvalid = min(self.bn, self.NB - n0) * self.bh * self.bw
        return tm, (n0 * self.H + h0) * self.W + w0, nvalid, tn


def plan_family(case, units):
    """The instantiation label tng_gemm_plan gives `case` over its first `units` units (scratch outputs)."""
    rows, Ncols, dev = units * case.unit_rows, case.weight.shape[0], case.weight.device
    kw = dict(bias=case.bias, alpha=case.alpha, act=case.act, block_n=case.block_n)
    if case.rowvec is not None:
        kw["rowvec"] = case.rowvec[:units]
    if case.alias:
        kw["res"] = kw["out_f32"] = torch.zeros(rows, Ncols, device=dev)
    else:
        if case.res is not None:
            kw["res"] = case.res[:rows]
        kw["out_f32"] = torch.empty(rows, Ncols, device=dev)
    if case.want_bf16:
        kw["out_bf16"] = torch.empty(rows, Ncols, device=dev, dtype=torch.bfloat16)
    W, NB = (units, 1) if case.linear else (case.W, units)
    if case.stats_hw:
        kw["gn_stats"], kw["stats_hw"] = torch.zeros(NB, Ncols, 2, dtype=torch.float64, device=dev), case.stats_hw
    return gemm_plan_family(slice_views(case.views, case.linear, 0, units), case.groups, case.weight, W, case.H, NB,
                            **kw)


def tall_schedule(case, sms):
    fam = plan_family(case, case.units)
    assert fam == "gemm_tc<160,m256>", fam
    sched = TallSchedule(case.W, case.H, case.NB, case.weight.shape[0], 160, 256, sms)
    case.block_n = 160
    # slices of SLICE_ROWS rows plan 128-row tiles, at most one work item per CTA
    per = SLICE_ROWS // case.unit_rows
    case.slices = lambda *_: [(a, min(a + per, case.units)) for a in range(0, case.units, per)]
    for units in {b - a for a, b in case.slices()}:
        assert plan_family(case, units) == "gemm_tc<160>"
        assert -(-units * case.unit_rows // 128) * sched.n_tiles <= sms
    return sched


def conv_case(g, cuda, NB, H, W, chans, Cout, *, stats=True):
    """3x3 convolution over a skip concatenation with bias, per-image vector, fp32 residual, fused GroupNorm
    statistics and fp32 + SiLU bf16 outputs (the resnet conv of the UNet's up path)."""
    a0s = (16, 8)[:len(chans)]
    views, data = skip_concat(g, cuda, NB, H, W, chans, a0s)
    groups, _ = skip_concat_groups(chans, a0s)
    Cs = sum(chans)
    wt = bf(rand(g, Cout, Cs, 3, 3, scale=(9 * Cs) ** -0.5))
    wk = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cs)
    res = poisoned(rand(g, NB * H * W, Cout).to(cuda))
    case = GemmCase(views, groups, poisoned(wk.to(cuda), col_pad=8, row_pad=0), W, H, NB, linear=False,
                    bias=rand(g, Cout).to(cuda), rowvec=rand(g, NB, Cout, scale=2.0).to(cuda), res=res,
                    act=L.ACT_SILU, stats_hw=H * W if stats else 0)
    case.want_bf16 = True
    return case, data, wk, res


def run_conv(cuda, case, data, wk, res):
    sms = num_sms()
    sched = tall_schedule(case, sms)
    assert all(sched.item(t)[2] == 256 for t in range(sched.work))    # full tiles: the fused-statistics epilogue
    NB, H, W, Cout = case.NB, case.H, case.W, case.weight.shape[0]
    rows = NB * H * W
    make = lambda: (Out(rows, Cout, dtype=torch.float32, device=cuda),
                    Out(rows, Cout, dtype=torch.bfloat16, device=cuda),
                    torch.zeros(NB, Cout, 2, dtype=torch.float64, device=cuda))
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    of, ob, st = outs
    xc = torch.cat([d.double() for d in data], dim=1).view(NB, H, W, -1)
    rs = sched.sample_rows(cuda)
    y, ab = gemm_rows_reference(xc, rs, TAPS3, wk.to(cuda), HW=H * W, bias=case.bias, rowvec=case.rowvec,
                                res=res.double())
    del xc
    sb = GEMM_GAMMA * ab
    e = excess_dev(of.hi[rs], y, sb + U32 * y.abs())
    z = act_ref(y, L.ACT_SILU)
    e = max(e, excess_dev(ob.hi[rs], z, 1.1 * sb + 2.0 ** -8 * z.abs()))
    # statistics = column sums of what was stored: fp32 partials over 16 rows, fp64 across partials
    o = of.hi.double().view(NB, H * W, Cout)
    sabs = o.abs().sum(1)
    e = max(e, excess_dev(st[..., 0], o.sum(1), 128 * U32 * sabs),
            excess_dev(st[..., 1], (o * o).sum(1), 128 * U32 * (o * o).sum(1)))
    assert e <= 1.0 and of.sentinel_intact() and ob.sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make, stats=torch.stack([sabs, (o * o).sum(1)], -1))
    return sched, e


def test_tall_tile_plan(cuda):
    """256 rows where the reduction is long and the launch has enough 256-row work items; 128 rows for the short-K
    linears and the level-0 320-channel convolution, for explicit N tiles other than 160 and for under-filled
    launches."""
    g = torch.Generator().manual_seed(40)

    def conv(NB, H, W, Cin, Cout, **kw):
        case, *_ = conv_case(g, cuda, NB, H, W, (Cin,), Cout, stats=False)
        for k, v in kw.items():
            setattr(case, k, v)
        return plan_family(case, NB)

    def linear(rows, Cin, Ncols, **kw):
        x = bf(rand(g, rows, Cin)).to(cuda)
        w = bf(rand(g, Ncols, Cin, scale=Cin ** -0.5)).to(cuda)
        case = GemmCase([row_view(x, 1, 1, rows)], [(0, 0, 0, 0, 0, (Cin + 63) // 64)], w, rows, 1, 1, linear=True,
                        **kw)
        return plan_family(case, rows)

    assert conv(16, 256, 16, 640, 320) == "gemm_tc<160,m256>"     # level 0, up path: K = 5760
    assert conv(16, 128, 8, 1280, 640) == "gemm_tc<160,m256>"     # level 1
    assert conv(16, 64, 4, 1280, 1280) == "gemm_tc<160,m256>"     # level 2: 128 work items
    assert conv(16, 256, 16, 320, 320) == "gemm_tc<160>"          # level 0, K = 2880
    assert conv(16, 256, 16, 640, 320, block_n=128) == "gemm_tc<128>"
    assert conv(2, 256, 16, 640, 320) == "gemm_tc<160>"           # 32 work items
    assert linear(65536, 320, 320) == "gemm_tc<160>"              # level-0 linears: K = 320 / 1280
    assert linear(65536, 1280, 320) == "gemm_tc<160>"
    assert linear(65536, 4096, 320) == "gemm_tc<160,m256>"


def test_tall_tile_resnet_conv_skip_concat(cuda):
    """Level-0 resnet conv 16 x 256 x 16 over a 320 + 320 skip concatenation -> 320: box 16 x 16 x 1."""
    g = torch.Generator().manual_seed(41)
    case, data, wk, res = conv_case(g, cuda, 16, 256, 16, (320, 320), 320)
    sched, e = run_conv(cuda, case, data, wk, res)
    assert (sched.bw, sched.bh, sched.bn) == (16, 16, 1) and sched.items_per_cta()[0] >= 3
    print(f"conv3x3 16x256x16 (320+320)->320 on 256-row tiles: {sched.work} work items; worst excess {e:.3f}")


def test_tall_tile_spans_images(cuda):
    """512 images of 8 x 4 pixels, 1280 -> 320 channels: one 256-row box (4 x 8 x 8) holds eight images, so the
    per-image vector and the GroupNorm statistics take the image of every warp's rows."""
    g = torch.Generator().manual_seed(42)
    case, data, wk, res = conv_case(g, cuda, 512, 8, 4, (1280,), 320)
    sched, e = run_conv(cuda, case, data, wk, res)
    assert (sched.bw, sched.bh, sched.bn) == (4, 8, 8)
    print(f"conv3x3 512x8x4 1280->320 on 256-row tiles spanning 8 images: worst excess {e:.3f}")


def test_tall_tile_ragged_rows_residual_aliases_output(cuda):
    """65436 rows (the last 256-row tile has 156) x 320, K = 4096, bias and alpha, with an fp32 residual that is the
    output: the predicated epilogue on both 64-row halves of the last tile, loads before stores."""
    sms = num_sms()
    g = torch.Generator().manual_seed(43)
    rows, Cin, Ncols = 65436, 4096, 320
    x = poisoned(bf(rand(g, rows, Cin)).to(cuda))
    wk = bf(rand(g, Ncols, Cin, scale=Cin ** -0.5))
    res0 = rand(g, rows, Ncols).to(cuda)
    case = GemmCase([row_view(x, 1, 1, rows)], [(0, 0, 0, 0, 0, Cin // 64)],
                    poisoned(wk.to(cuda), col_pad=8, row_pad=0), rows, 1, 1, linear=True,
                    bias=rand(g, Ncols).to(cuda), alias=True, alpha=0.75)
    sched = tall_schedule(case, sms)
    assert sched.item(sched.work - 1)[2] == rows % 256 > 64
    make = lambda: (Out(rows, Ncols, dtype=torch.float32, device=cuda, ld=Ncols + 8, init=res0), None, None)
    outs = make()
    case.launch(*outs)
    torch.cuda.synchronize()
    rs = sched.sample_rows(cuda)
    y, ab = gemm_rows_reference(x.double().view(1, 1, rows, Cin), rs, [(0, 0)], wk.to(cuda), HW=rows,
                                bias=case.bias, res=res0, alpha=case.alpha)
    e = excess_dev(outs[0].hi[rs], y, GEMM_GAMMA * ab + U32 * y.abs())
    assert e <= 1.0 and outs[0].sentinel_intact()
    check_sliced_and_repeat(case, sched, sms, outs, make)
    print(f"linear 65436x320 K=4096 on 256-row tiles, res == out: worst excess {e:.3f}")
