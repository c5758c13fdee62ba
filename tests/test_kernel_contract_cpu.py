"""CPU checks of the helpers in test_kernel_contract_gpu.py: the poisoned / sentinel buffers, the per-element error
metrics and the references must themselves be right, or the GPU contract tests prove nothing."""
import math

import torch
import torch.nn.functional as F

import cabi_spec as S
from tango_b200 import lib as L
from tango_b200 import ops
from test_kernel_contract_gpu import (FMIN, GEMM_GAMMA, NAN, SENT, U32, Out, attn_ref, bf, coef_rows, dpm_rows,
                                      el_err, excess, flat_base, gelu64, gemm_reference, geglu_linear_reference,
                                      geglu_operands, geglu_reference, geglu_weights, group_fit, k_groups_1x1,
                                      linear_f32_operands, linear_f32_reference, pack_split, poisoned, poisoned_flat,
                                      rel_attn_bound, rel_attn_kbias, rel_attn_operands, rel_attn_ref, row_view,
                                      rowcol_err, silu64, skip_concat, skip_concat_groups)


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


def catches(ref, bound, rel=2.0 ** -12) -> bool:
    """The bound is not vacuous: on most elements of at least rms size, a single element wrong by `rel` of itself
    exceeds its allowance (the rest are elements whose allowance is large for a reason, e.g. a GEGLU gate near 0)."""
    ref, bound = ref.double(), torch.as_tensor(bound).double()
    big = ref.abs() >= ref.pow(2).mean().sqrt()
    return bool(big.any()) and (rel * ref.abs()[big] > bound[big]).double().mean().item() > 0.5


def test_geglu_reference_matches_torch():
    """gelu64 equals F.gelu (both forms) over the gate range; through spec_conv_gemm, PackedConv's interleaved weights
    and bias give F.linear followed by hidden * gelu(gate); the per-element allowances are not vacuous."""
    x = torch.linspace(-9.0, 9.0, 3601, dtype=torch.float64)
    for tanh in (False, True):
        assert torch.allclose(gelu64(x, tanh), F.gelu(x, approximate="tanh" if tanh else "none"), rtol=1e-12, atol=1e-13)
    u = math.sqrt(2.0 / math.pi) * (10.0 + 0.044715 * 1000.0)   # the tail keeps its digits: -10 e^(-2u) (1 + O(e^-2u))
    assert abs(gelu64(torch.tensor([-10.0]), True).item() / (-10.0 * math.exp(-2.0 * u)) - 1.0) < 1e-12
    g = torch.Generator().manual_seed(11)
    rows, Cin, inner = 40, 128, 256
    xr = torch.randn(rows, Cin, generator=g)
    wt, b = geglu_weights(g, 2 * inner, 2 * inner, Cin)
    for tanh in (False, True):
        pc = ops.PackedConv(wt, b, split=True, device="cpu", geglu_bn=256, geglu_tanh=tanh)
        xin = torch.cat(pack_split(xr), dim=1)      # dense: the spec reads a view's tensor as its storage
        ob = Out(rows, inner, dtype=torch.bfloat16, device="cpu", split_off=inner, ld=2 * inner)
        S.spec_conv_gemm(ops.act_views(xin, 1, 1, rows, Cin, True), pc.groups(), pc.weight, rows, 1, 1, bias=pc.bias,
                         out_bf16=ob.view, act=L.ACT_GEGLU_TANH if tanh else L.ACT_GEGLU, split_off=inner, block_n=256)
        z, bound = geglu_linear_reference(xr, wt, b, tanh, gamma=2 * GEMM_GAMMA)
        bound = bound + 2.0 ** -16 * z.abs()
        assert excess(ob.value(), z, bound) <= 1.0 and ob.sentinel_intact()
        assert catches(z, bound)
        # the interleave matters: hidden and gate swapped is far outside the bound
        y = F.linear(xr.double(), wt.double(), b.double())
        assert excess(y[:, inner:] * gelu64(y[:, :inner], tanh), z, bound) > 1e3
    # the GPU test's operands: the gates span both tails, and the bound of its hi + lo check is not vacuous
    for bn in (128, 256):
        x, w, bias = geglu_operands(g, "cpu", 300, bn)
        views, groups = [row_view(x, 1, 1, 300)], k_groups_1x1(x.shape[1])
        y, absdot = gemm_reference(views, groups, w, 300, 1, 1, bias=bias)
        for tanh in (False, True):
            z, bound = geglu_reference(y, absdot, bn, tanh)
            assert catches(z, bound + 2.0 ** -16 * z.abs())


def t5_attention_loops(q, k, v, relbias, kbias, B, heads, L_):
    """T5Attention written out per (batch, head, query): scores = q . k + relbias[h, key - query + L - 1] + mask, no
    scaling, softmax over the keys, weighted sum of the values."""
    out = torch.zeros(B * L_, heads * 64, dtype=torch.float64)
    for b in range(B):
        for h in range(heads):
            cs = slice(64 * h, 64 * h + 64)
            K, V = k[b * L_:(b + 1) * L_, cs].double(), v[b * L_:(b + 1) * L_, cs].double()
            for i in range(L_):
                s = K @ q[b * L_ + i, cs].double()
                s = s + torch.stack([relbias[h, j - i + L_ - 1].double() for j in range(L_)])
                if kbias is not None:
                    s = s + kbias[b].double()
                e = torch.exp(s - s.max())
                out[b * L_ + i, cs] = (e / e.sum()) @ V
    return out


def test_rel_attention_reference_matches_t5_formula():
    """The fp64 rel-attention reference equals T5Attention written out, and the fp32 spec statement; a fully masked
    sequence is the uniform mean of its values; the allowance is not vacuous."""
    g = torch.Generator().manual_seed(6)
    for mask in (None, "tail", "all but key 0", "one sequence"):
        B, heads, L_ = 3, 2, 7
        q, k, v, relbias = rel_attn_operands(g, B, heads, L_)
        kb = rel_attn_kbias(B, L_, mask)
        ref, pv, ds = rel_attn_ref(q, k, v, relbias, kb, batch=B, heads=heads, L=L_)
        assert el_err(ref, t5_attention_loops(q, k, v, relbias, kb, B, heads, L_)) < 1e-12
        qkv = torch.cat([q, k, v], dim=1)
        o = torch.zeros(B * L_, heads * 64, dtype=torch.bfloat16)
        S.spec_rel_attention(qkv, relbias, kb, o, batch=B, heads=heads, L=L_, q_col0=0, k_col0=heads * 64,
                             v_col0=2 * heads * 64)
        assert el_err(o, ref) < 2.0 ** -6                  # bf16 output
        if mask == "one sequence":
            assert el_err(ref.view(B, L_, -1)[1], v.double().view(B, L_, -1)[1].mean(0).expand(L_, -1)) < 1e-12
        if mask is None:
            assert catches(ref, rel_attn_bound(pv, ds, L_) + 2.0 ** -16 * ref.abs())
    q, k, v, relbias = rel_attn_operands(g, 2, 16, 65)
    ref, pv, ds = rel_attn_ref(q, k, v, relbias, None, batch=2, heads=16, L=65)
    assert catches(ref, rel_attn_bound(pv, ds, 65) + 2.0 ** -16 * ref.abs())
    assert FMIN + 30.0 == FMIN and torch.tensor(FMIN) + 30.0 == torch.tensor(FMIN)   # both absorb the scores


def test_linear_f32_reference_and_bound():
    g = torch.Generator().manual_seed(8)
    for pre in (L.ACT_NONE, L.ACT_SILU):
        for post in (L.ACT_NONE, L.ACT_SILU):
            x, w, b = linear_f32_operands(g, "cpu", 5, 320, 1280, True)
            ref, bound = linear_f32_reference(x, w, b, pre, post)
            a = F.silu(x.double()) if pre else x.double()
            want = F.linear(a, w.double(), b.double())
            assert el_err(ref, F.silu(want) if post else want) < 1e-14
            assert torch.equal(silu64(x.double()), x.double() * torch.sigmoid(x.double()))
            assert catches(ref, bound)


def test_dpm_rows_cover_every_order():
    rows = dpm_rows()
    assert len(rows) == 12 and [o for _, o, _ in rows] == [1, 2, 3] * 4
    assert all(r.shape == (11,) and torch.isfinite(r).all() for _, _, r in rows)
    assert all(float(r[9]) != float(r[10]) for _, o, r in rows if o == 3)   # w_r and 1/(r0 + r1) differ
