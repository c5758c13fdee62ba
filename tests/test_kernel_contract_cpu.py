"""CPU checks of the helpers in test_kernel_contract_gpu.py: the poisoned / sentinel buffers, the per-element error
metrics and the references must themselves be right, or the GPU contract tests prove nothing."""
import math

import torch
import torch.nn.functional as F

from tango_b200 import ops
from test_kernel_contract_gpu import (NAN, SENT, U32, Out, attn_ref, bf, coef_rows, el_err, excess,
                                      flat_base, gemm_reference, group_fit, poisoned, poisoned_flat, rowcol_err,
                                      skip_concat, skip_concat_groups)


def test_poisoned_buffers_and_sentinels():
    t = torch.arange(12.0).view(3, 4)
    v = poisoned(t, col0=2, col_pad=3, align=8)
    assert torch.equal(v, t) and v.stride(0) % 8 == 0 and v.stride(0) >= 2 + 4 + 3
    base = flat_base(v)
    assert base.numel() == (3 + 3) * v.stride(0) - 2 and torch.isnan(base[4:v.stride(0)]).all()
    f = poisoned_flat(torch.ones(5), lead=3)
    assert f.storage_offset() == 3 and torch.isnan(flat_base(f)[5:]).all()
    for dt in (torch.float32, torch.bfloat16):
        o = Out(4, 3, dtype=dt, device="cpu", col0=1, split_off=5, ld=12)
        assert torch.isnan(o.hi).all() and torch.isnan(o.lo).all() and o.sentinel_intact()
        assert (o.buf[:4, 4:6] == SENT).all() and (o.buf[4:] == SENT).all()
        o.hi.fill_(1.0)
        o.lo.fill_(0.0)
        assert o.sentinel_intact() and el_err(o.value(), torch.ones(4, 3)) == 0.0
        o.hi[2, 1] = NAN                                          # an element the kernel never wrote
        assert el_err(o.value(), torch.ones(4, 3)) == math.inf
        o.hi[2, 1] = 1.0
        o.buf[1, 4] = SENT + 1                                    # a stray write between the halves
        assert not o.sentinel_intact()
        o.buf[1, 4] = SENT
        o.buf[4, 0] = -0.0 if dt == torch.float32 else SENT       # past the last row (a sign flip counts too)
        o.buf[5, 11] = NAN
        assert not o.sentinel_intact()


def test_error_metrics_see_one_bad_element():
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(512, 96, generator=g, dtype=torch.float64)
    got = ref + 1e-9 * torch.randn(512, 96, generator=g, dtype=torch.float64)
    assert el_err(got, ref) < 1e-8 and rowcol_err(got, ref) < 1e-7
    assert excess(got, ref, 1e-8 + 0 * ref) <= 1.0
    bad = got.clone()
    bad[300, 17] += 1e-4                                          # one element, 1e-4 of the rms: a Frobenius error of ~5e-7
    assert el_err(bad, ref) > 9e-5 and excess(bad, ref, 1e-8 + 0 * ref) > 1e3
    assert ((bad - ref).norm() / ref.norm()).item() < 1e-6
    small = ref.clone()
    small[7] *= 1e-2                                              # a small row, wrong by 10 % of its own size
    bad = small.clone()
    bad[7] *= 1.1
    assert el_err(bad, small) < 1e-2 and rowcol_err(bad, small) > 5e-2


def test_gemm_reference_matches_conv2d():
    """The spec-driven GEMM reference on the poisoned multi-view skip-concat layout equals F.conv2d of the concatenation,
    and the |operand| contraction bounds it."""
    g = torch.Generator().manual_seed(1)
    chans, a0s = (72, 200, 64), (16, 24, 8)
    NB, H, W, Cout = 2, 4, 8, 24
    views, data = skip_concat(g, "cpu", NB, H, W, chans, a0s)
    groups, Ktot = skip_concat_groups(chans, a0s)
    Cs = sum(chans)
    wt = bf(torch.randn(Cout, Cs, 3, 3, generator=g) / math.sqrt(9 * Cs))
    w = poisoned(wt.permute(0, 2, 3, 1).reshape(Cout, Ktot), col_pad=8, row_pad=0)
    bias = torch.randn(Cout, generator=g)
    y, absdot = gemm_reference(views, groups, w, W, H, NB, bias=bias, alpha=0.5)
    xc = torch.cat([d.double() for d in data], dim=1).view(NB, H, W, Cs).permute(0, 3, 1, 2)
    ref = (F.conv2d(xc, wt.double(), bias.double(), padding=1) * 0.5).permute(0, 2, 3, 1).reshape(-1, Cout)
    assert excess(y, ref, 2 * U32 * ref.abs() + 1e-30) <= 1.0
    assert (absdot.double() >= ref.abs() * (1 - 1e-6)).all() and torch.isfinite(absdot).all()
    # a wrong a_c0 reads the NaN channels in front of the data: the reference would see them
    bad = [(v, a0 - 8, dw, dh, bk, n) for (v, a0, dw, dh, bk, n) in groups]
    y2, _ = gemm_reference(views, bad, w, W, H, NB, bias=bias, alpha=0.5)
    assert not torch.isfinite(y2).all()


def test_stride2_references_match_torch():
    """The stride-2 parity views + k-groups, through the spec, equal F.conv2d on odd H / W for padding 1 and for the
    padding-0 form with the bottom / right zero fill the GPU test builds with F.pad; the rowvec / residual epilogue."""
    g = torch.Generator().manual_seed(2)
    NB, H, W, Cin, Cout = 2, 9, 7, 64, 16
    x = bf(torch.randn(NB, Cin, H, W, generator=g))
    wt = bf(torch.randn(Cout, Cin, 3, 3, generator=g) / 24)
    rows = poisoned(x.permute(0, 2, 3, 1).reshape(-1, Cin))
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    rv = torch.randn(NB, Cout, generator=g)
    res = torch.randn(NB * Ho * Wo, Cout, generator=g)
    for pad in (1, 0):
        pc = ops.PackedConv(wt.float(), None, split=False, device="cpu", stride=2, pad=pad)
        views = ops.parity_views(rows, NB, H, W, Cin, False)
        y, _ = gemm_reference(views, pc.groups(parity_views=[0, 1, 2, 3]), pc.weight, Wo, Ho, NB, rowvec=rv, res=res)
        xr = x.double() if pad else F.pad(x.double(), (0, 2 * Wo + 1 - W, 0, 2 * Ho + 1 - H))
        ref = F.conv2d(xr, wt.double(), stride=2, padding=pad) + rv.double()[:, :, None, None]
        ref = ref.permute(0, 2, 3, 1).reshape(-1, Cout) + res.double()
        assert excess(y, ref, 2 * U32 * ref.abs() + 1e-30) <= 1.0


def test_attention_reference_matches_torch():
    g = torch.Generator().manual_seed(3)
    B, heads, Lq, Lk = 2, 3, 5, 9
    q, k, v = (torch.randn(B * n, heads * 64, generator=g, dtype=torch.float64) for n in (Lq, Lk, Lk))
    kb = torch.zeros(B, Lk)
    kb[1, 4:] = -10000.0
    o, pv = attn_ref(q, k, v, batch=B, heads=heads, Lq=Lq, Lk=Lk, scale=0.125, kbias=kb)
    sh = lambda t, n: t.view(B, n, heads, 64).transpose(1, 2)
    ref = F.scaled_dot_product_attention(sh(q, Lq), sh(k, Lk), sh(v, Lk), attn_mask=kb.double()[:, None, None, :],
                                         scale=0.125).transpose(1, 2).reshape(B * Lq, -1)
    assert el_err(o, ref) < 1e-12
    assert (pv >= o.abs() - 1e-12).all()


def test_groupnorm_fit_and_sched_rows():
    g = torch.Generator().manual_seed(4)
    NB, HW, Cc, groups = 2, 64, 32, 4
    x = torch.randn(NB, Cc, HW, generator=g, dtype=torch.float64) * 3 + 40
    ref = F.group_norm(x, groups).permute(0, 2, 1).reshape(NB * HW, Cc)
    da, db, resid = group_fit(ref * (1 + 3e-5) + 2e-5, ref, NB, HW, groups)
    assert abs(da - 3e-5) < 1e-9 and abs(db - 2e-5) < 1e-9 and resid < 1e-12
    rows = dict(coef_rows())
    assert rows["ddpm-eps-clip"][8] > 0 and all(float(r[8]) == 0 for n, r in rows.items() if n != "ddpm-eps-clip")
    assert float(rows["ddpm-eps-clip"][4]) != 0            # a mid-schedule DDPM row draws noise
    assert float(rows["ddim-eps"][7]) != 0 and not torch.equal(rows["ddim-eps"], rows["ddim-v"])
