"""CPU checks of the helpers in test_kernels_at_scale_gpu.py: the row-sampled GEMM reference, the work-item schedule
mirrors and the per-batch attention reference must themselves be right, or the GPU cases prove nothing."""
import torch
import torch.nn.functional as F

from tango_b200 import lib as L
from test_kernel_contract_gpu import attn_ref, gemm_reference, k_groups_1x1, row_view
from test_kernels_at_scale_gpu import (TAPS3, GemmSchedule, excess_dev, gemm_rows_reference, gn_apply_batches, gn_slab,
                                       im2col_rows, same_bits, slice_views)


def test_im2col_rows_reference_matches_conv2d():
    """The sampled 3x3 'same' convolution (taps in the packed tap-major order, zero outside each image) equals
    F.conv2d at every sampled row, including rows on every image border; the |operand| pass equals the conv of |x|."""
    g = torch.Generator().manual_seed(0)
    NB, H, W, C, Cout = 3, 5, 4, 6, 7
    x = torch.randn(NB, C, H, W, generator=g, dtype=torch.float64)
    wt = torch.randn(Cout, C, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(Cout, generator=g, dtype=torch.float64)
    rv = torch.randn(NB, Cout, generator=g, dtype=torch.float64)
    res = torch.randn(NB * H * W, Cout, generator=g, dtype=torch.float64)
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(-1, Cout)
    full = nhwc(F.conv2d(x, wt, b, padding=1) + rv[:, :, None, None]) + res
    fabs = nhwc(F.conv2d(x.abs(), wt.abs(), b.abs(), padding=1) + rv.abs()[:, :, None, None]) + res.abs()
    rows = torch.tensor([0, 3, 4, 19, 20, 37, 59])
    wk = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * C)
    y, ab = gemm_rows_reference(x.permute(0, 2, 3, 1), rows, TAPS3, wk, HW=H * W, bias=b, rowvec=rv, res=res,
                                alpha=-0.5)
    assert torch.allclose(y, -0.5 * full[rows], rtol=1e-12, atol=1e-12)
    assert torch.allclose(ab, 0.5 * fabs[rows], rtol=1e-12, atol=1e-12)
    assert im2col_rows(x.permute(0, 2, 3, 1), rows, TAPS3).shape == (len(rows), 9 * C)


def test_linear_rows_reference_matches_spec():
    """The linear form (rows on the W axis, one tap) equals cabi_spec.spec_conv_gemm on the same bf16 operands."""
    g = torch.Generator().manual_seed(1)
    rows, Cin, Ncols = 300, 72, 40
    x = torch.randn(rows, Cin, generator=g).to(torch.bfloat16)
    w = torch.randn(Ncols, Cin, generator=g).to(torch.bfloat16)
    bias, res = torch.randn(Ncols, generator=g), torch.randn(rows, Ncols, generator=g)
    y_spec, ab_spec = gemm_reference([row_view(x, 1, 1, rows)], k_groups_1x1(Cin), w, rows, 1, 1, bias=bias, res=res,
                                     alpha=0.75)
    rs = torch.arange(rows)
    y, ab = gemm_rows_reference(x.double().view(1, 1, rows, Cin), rs, [(0, 0)], w, HW=rows, bias=bias, res=res,
                                alpha=0.75)
    assert torch.allclose(y, y_spec.double(), rtol=1e-5, atol=1e-5)      # the spec accumulates in fp32
    assert torch.allclose(ab, ab_spec.double(), rtol=1e-5, atol=1e-5)


def test_slice_views_address_the_same_elements():
    """A sliced view (rows of a linear, images of a convolution) reads exactly the rows the whole view has there."""
    t = torch.arange(40 * 24, dtype=torch.float32).view(40, 24).to(torch.bfloat16)
    lin = slice_views([row_view(t[:, 8:], 1, 1, 40)], True, 10, 25)[0]
    assert (lin.W, lin.H, lin.NB) == (15, 1, 1)
    first = lambda v: t.view(-1)[v.t.storage_offset() + v.off]               # the element the view's pointer names
    assert first(lin) == t[10, 8]
    conv = slice_views([L.View(t, 16, 4, 2, 5, 24, 4 * 24, 8 * 24, off=8)], False, 2, 4)[0]
    assert (conv.W, conv.H, conv.NB) == (4, 2, 2) and first(conv) == t[2 * 8, 8]


def test_gemm_schedule_mirrors_the_host_tiling():
    """M tiling of plan_gemm at the UNet shapes: 65536-row linears and the 16 x 256 x 16 conv are 512 M tiles; the
    32 x 2 level is 8 tiles of two images (the under-filled launch the kernel's comment names); rows of a tile are a
    prefix of consecutive output rows and every row lies in exactly one tile."""
    for W, H, NB, m_tiles, bw_bh_bn in [(65536, 1, 1, 512, (128, 1, 1)), (16, 256, 16, 512, (16, 8, 1)),
                                        (2, 32, 16, 8, (2, 32, 2)), (4, 2, 13, 1, (4, 2, 16)),
                                        (30000, 1, 1, 235, (128, 1, 1))]:
        s = GemmSchedule(W, H, NB, 320, 160, 1, 132)
        assert s.m_tiles == m_tiles and (s.bw, s.bh, s.bn) == bw_bh_bn
        covered = torch.zeros(W * H * NB, dtype=torch.int32)
        for tm in range(s.m_tiles):
            _, r0, nvalid, tn = s.item(tm * s.n_tiles)
            assert tn == 0 and 0 < nvalid <= 128
            covered[r0:r0 + nvalid] += 1
        assert (covered == 1).all()


def test_gemm_sample_covers_every_work_item_position():
    """The sampled rows contain every work item of the sampled CTAs (every index j of their sequences, whichever N
    tile it is) and the last M tile; on 132 and on 114 SMs."""
    for sms in (132, 114):
        s = GemmSchedule(30000, 1, 1, 584, 128, 1, sms)
        rows = set(s.sample_rows().tolist())
        assert max(rows) == 29999 and 0 in rows
        for c in s.sample_ctas():
            seq = s.sequence(c)
            assert len(seq) >= s.items_per_cta()[0] >= 3
            for t in seq:
                _, r0, nvalid, _ = s.item(t)
                assert set(range(r0, r0 + nvalid)) <= rows
        shapes = {s.epilogue(t) for c in range(s.grid) for t in s.sequence(c)}
        assert shapes == {"full", "partial-n", "partial-m"}


def test_gn_apply_batches_mirror():
    """gn_slab mirrors tng_groupnorm_apply's slab choice; gn_apply_batches splits every thread's rows into balanced
    batches of at most 8 whose sizes add up to the image's rows."""
    assert gn_slab(960, 32) == (240, 4) and gn_slab(320, 32) == (320, 1) and gn_slab(2560, 32) == (320, 8)
    for C, HW in ((960, 4096), (320, 4096), (2560, 64), (320, 37)):
        slab = gn_slab(C, 32)[0]
        RL = 256 // min(slab // 4, 256)
        for per_sm in (1, 3, 8):
            bt = gn_apply_batches(16, HW, C, 32, per_sm, 132)
            assert all(per <= 8 and 0 < last <= per for _, per, last in bt)
            assert sum((nb - 1) * per + last for nb, per, last in bt) == HW    # each row of an image once
            assert len(bt) <= RL * HW


def test_per_batch_attention_reference_matches_sdpa():
    """attn_ref on one batch entry (as the GPU cases call it) equals F.scaled_dot_product_attention with the same
    additive key mask."""
    g = torch.Generator().manual_seed(3)
    B, heads, Lq, Lk = 2, 3, 37, 70
    q = torch.randn(B * Lq, heads * 64, generator=g, dtype=torch.float64)
    k = torch.randn(B * Lk, heads * 64, generator=g, dtype=torch.float64)
    v = torch.randn(B * Lk, heads * 64, generator=g, dtype=torch.float64)
    kb = torch.zeros(B, Lk, dtype=torch.float64)
    kb[1, 50:] = -10000.0
    for b in range(B):
        rq, rk = slice(b * Lq, (b + 1) * Lq), slice(b * Lk, (b + 1) * Lk)
        ref, pv = attn_ref(q[rq], k[rk], v[rk], batch=1, heads=heads, Lq=Lq, Lk=Lk, scale=0.125, kbias=kb[b:b + 1])
        hd = lambda t, n: t.view(n, heads, 64).transpose(0, 1)
        want = F.scaled_dot_product_attention(hd(q[rq], Lq), hd(k[rk], Lk), hd(v[rk], Lk),
                                              attn_mask=kb[b].view(1, 1, Lk), scale=0.125)
        assert torch.allclose(ref, want.transpose(0, 1).reshape(Lq, -1), rtol=1e-10, atol=1e-12)
        assert (pv >= ref.abs() - 1e-12).all()


def test_bit_and_excess_helpers():
    a = torch.tensor([0.0, 1.0, float("nan")])
    assert same_bits(a, a.clone()) and not same_bits(a, torch.tensor([-0.0, 1.0, float("nan")]))
    ref = torch.tensor([1.0, 2.0])
    assert excess_dev(torch.tensor([1.5, 2.0]), ref, torch.tensor([1.0, 1.0])) == 0.5
    assert excess_dev(torch.tensor([1.0, float("inf")]), ref, torch.tensor([1.0, 1.0])) == float("inf")
