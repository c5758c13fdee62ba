"""GPU: each C-ABI entry point against its `cabi_spec` statement (or an fp64 torch evaluation of the same bf16-rounded
operands) at the descriptor features the host actually uses: sliced and offset operands, ld > C, ragged tails, several
images per tile, scalar (misaligned / Ncols % 4 != 0) epilogues, hi/lo outputs, aliasing; the GEGLU epilogue, the T5
and mel front ends and the DPM-Solver step at the layouts the generate and edit paths use.

Every input is a view into a larger buffer whose padding holds NaN, so a read past the logical extent poisons the result.
Every output starts as NaN in its logical region (an element the kernel never writes fails) and as a finite sentinel
everywhere else: between the hi and lo halves, past ld and past the last row. The sentinel must survive bit for bit.
Errors are measured per element (`el_err`, `excess`), so a single bad row, column or tile cannot hide in a norm."""
from __future__ import annotations

import math

import pytest
import torch
import torch.nn.functional as F

import cabi_spec as S
from tango_b200 import lib as L
from tango_b200 import ops
from tango_b200.schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler

pytestmark = pytest.mark.gpu

NAN = float("nan")
SENT = -7.0       # output padding sentinel: exact in fp32 and bf16
U32 = 2.0 ** -24  # fp32 unit round-off
# per-element GEMM allowance relative to sum |a_k b_k| (+ |epilogue terms|): fp32 accumulation over K <= ~1.2k products
# has a typical relative error ~ sqrt(K) * 2^-24 <= 2^-19; 2^-16 leaves an 8x margin and still sees a single wrong
# product of a normal-sized operand
GEMM_GAMMA = 2.0 ** -16


def gemm_gamma(k: int) -> float:
    """GEMM_GAMMA for a reduction of k products, long ones included. The sqrt(k) argument above needs products of
    random sign; a sum whose products share their sign (softmax P times a value column with a non-zero mean: the
    split-mode VAE attention, K = 3 x 4096) grows its partial sums steadily, and so does the rounding error. Worst case:
    wgmma adds one k-step of 16 products to the fp32 accumulator per instruction, and an update rounded in either
    direction (the tensor core need not round to nearest) errs by at most one ulp, 2u of a partial sum whose magnitude is
    at most sum |a_k b_k|: (k / 16) * 2^-23 = k * 2^-27 of that sum. Below k = 2048 that is within GEMM_GAMMA; the
    UNet's 1280-channel 3 x 3 convolution (k = 11 520) gets 2^-13.5, its split form (3 x 11 520) 2^-11.9. On an H100
    80GB HBM3 (700 W power limit) the k = 12 288 P V product exceeds the fixed 2^-16 bound by a factor of 1.22."""
    return max(GEMM_GAMMA, k * 2.0 ** -27)


def bf(x):
    return x.to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------- buffers
def poisoned(t: torch.Tensor, *, col0: int = 0, col_pad: int = 8, row_pad: int = 3, align: int = 8) -> torch.Tensor:
    """t [R, C] copied into a NaN-filled [R + row_pad, ld] buffer at column col0 (ld a multiple of `align`, >= col0 + C +
    col_pad); returns the [R, C] view (its stride(0) is the buffer's ld)."""
    R, C = t.shape
    ld = col0 + C + col_pad
    ld += (-ld) % align
    buf = torch.full((R + row_pad, ld), NAN, dtype=t.dtype, device=t.device)
    v = buf[:R, col0:col0 + C]
    v.copy_(t)
    return v


def poisoned_flat(t: torch.Tensor, *, lead: int = 0, tail: int = 16) -> torch.Tensor:
    """1-D NaN-padded copy of t starting `lead` elements into its buffer."""
    buf = torch.full((lead + t.numel() + tail,), NAN, dtype=t.dtype, device=t.device)
    v = buf[lead:lead + t.numel()]
    v.copy_(t.reshape(-1))
    return v


class Out:
    """Output buffer [rows + row_pad, ld]: the logical columns [col0, col0 + cols) (and, when split_off > 0, the lo half at
    col0 + split_off) start as NaN, every other element holds the sentinel."""

    def __init__(self, rows, cols, *, dtype, device, ld=None, col0=0, split_off=0, row_pad=2, init=None):
        ld = ld if ld is not None else col0 + max(cols, split_off + cols if split_off else cols) + 8
        assert ld >= col0 + (split_off if split_off else 0) + cols
        self.rows, self.cols, self.col0, self.split_off = rows, cols, col0, split_off
        self.buf = torch.full((rows + row_pad, ld), SENT, dtype=dtype, device=device)
        self.mask = torch.zeros(self.buf.shape, dtype=torch.bool, device=device)
        self.mask[:rows, col0:col0 + cols] = True
        if split_off:
            self.mask[:rows, col0 + split_off:col0 + split_off + cols] = True
        self.buf[self.mask] = NAN
        if init is not None:
            self.hi.copy_(init)

    @property
    def view(self):      # what the kernel gets: pointer at col0, ld = the buffer's row stride
        return self.buf[:self.rows, self.col0:]

    @property
    def hi(self):
        return self.buf[:self.rows, self.col0:self.col0 + self.cols]

    @property
    def lo(self):
        return self.buf[:self.rows, self.col0 + self.split_off:self.col0 + self.split_off + self.cols]

    def value(self):     # hi + lo (fp64), or just the stored value
        v = self.hi.double()
        return v + self.lo.double() if self.split_off else v

    def cpu_clone(self):
        o = Out.__new__(Out)
        o.__dict__.update(self.__dict__)
        o.buf, o.mask = self.buf.cpu().clone(), self.mask.cpu()
        return o

    def sentinel_intact(self) -> bool:
        out = self.buf[~self.mask]
        bits = torch.int16 if self.buf.element_size() == 2 else torch.int32
        want = torch.tensor([SENT], dtype=self.buf.dtype).view(bits).item()
        return bool((self.buf.view(bits)[~self.mask] == want).all().item()) and out.numel() > 0


# ---------------------------------------------------------------------------------------------------- error metrics
def el_err(got, ref) -> float:
    """max |got - ref| / rms(ref) over elements (inf if got has a NaN / inf): a single bad element decides."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    if not torch.isfinite(got).all():
        return math.inf
    rms = ref.pow(2).mean().sqrt().clamp_min(1e-30)
    return ((got - ref).abs().max() / rms).item()


def rowcol_err(got, ref) -> float:
    """el_err per row and per column (each normalised by its own rms, floored at 1e-2 of the global rms): a bad row or
    column of small magnitude cannot hide behind large ones."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    if not torch.isfinite(got).all():
        return math.inf
    d = (got - ref).abs()
    floor = 1e-2 * ref.pow(2).mean().sqrt().clamp_min(1e-30)
    r = (d.amax(1) / ref.pow(2).mean(1).sqrt().clamp_min(floor)).max()
    c = (d.amax(0) / ref.pow(2).mean(0).sqrt().clamp_min(floor)).max()
    return max(r.item(), c.item())


def excess(got, ref, bound) -> float:
    """max |got - ref| / bound over elements (<= 1 passes; inf on NaN / inf); bound is a per-element allowance."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    if not torch.isfinite(got).all():
        return math.inf
    b = torch.as_tensor(bound, dtype=torch.float64).cpu().clamp_min(1e-300)
    return ((got - ref).abs() / b).max().item()


# ---------------------------------------------------------------------------------------------------- GEMM harness
def flat_base(t):
    """1-D tensor over t's storage from t's first element to the end of the allocation (the memory a view's strides and
    offset address)."""
    n = t.untyped_storage().nbytes() // t.element_size() - t.storage_offset()
    return t.as_strided((n,), (1,))


def _cpu_view(v, f=None):
    return L.View(_cpu(flat_base(v.t), f), v.C, v.W, v.H, v.NB, v.s_w, v.s_h, v.s_n, v.off)


def _cpu(x, f=None):
    if x is None:
        return None
    x = x.detach().cpu()
    return f(x) if f is not None else x


def gemm_reference(views, groups, weight, W, H, NB, *, prior=None, **kw):
    """spec_conv_gemm on CPU copies -> (y fp32 [rows, Ncols], absdot [rows, Ncols]); absdot = the same contraction and
    epilogue on |operands| (the per-element scale of the fp32 summation error)."""
    rows, Ncols = NB * H * W, weight.shape[0]
    res_out = []
    for f in (None, torch.abs):
        vs = [_cpu_view(v, f) for v in views]
        ek = {k: _cpu(kw[k], f) for k in ("bias", "rowvec", "res") if kw.get(k) is not None}
        out = torch.zeros(rows, Ncols) if prior is None else _cpu(prior, f).float().clone()
        alpha = kw.get("alpha", 1.0)
        S.spec_conv_gemm(vs, groups, _cpu(weight, f), W, H, NB, alpha=abs(alpha) if f else alpha,
                         accumulate=prior is not None, rowvec_ld=kw.get("rowvec_ld", 0), out_f32=out, **ek)
        res_out.append(out)
    return res_out[0], res_out[1]


def act_ref(y, act, act_param=0.0):
    y = y.double()
    if act == L.ACT_SILU:
        return F.silu(y)
    if act == L.ACT_LRELU:
        return F.leaky_relu(y, act_param)
    return y


def gemm_plan_family(views, groups, weight, W, H, NB, **kw) -> str:
    """The instantiation tng_gemm_plan picks for this descriptor (as the profiler labels it)."""
    L.PROF.start()
    try:
        L.conv_gemm(views, groups, weight, W, H, NB, **kw)
    finally:
        fams = L.PROF.stop()
    assert len(fams) == 1
    return next(iter(fams))


def check_gemm(views, groups, weight, W, H, NB, *, of=None, ob=None, act=L.ACT_NONE, act_param=0.0, prior=None,
               gamma=GEMM_GAMMA, **kw):
    """Launch tng_conv_gemm into the Out buffers of/ob and hold every element to the spec: fp32 output within the
    summation bound, bf16 output within bf16 rounding (hi: 2^-8 relative, hi+lo: 2^-16) of act(y), sentinels intact."""
    kw.pop("accumulate", None)
    y, absdot = gemm_reference(views, groups, weight, W, H, NB, prior=prior, **kw)
    L.conv_gemm(views, groups, weight, W, H, NB, accumulate=prior is not None, out_f32=None if of is None else of.view,
                out_bf16=None if ob is None else ob.view, act=act, act_param=act_param,
                split_off=0 if ob is None else ob.split_off, **kw)
    torch.cuda.synchronize()
    sum_bound = gamma * absdot.double() + 1e-30
    if of is not None:
        assert excess(of.hi, y, sum_bound + U32 * y.double().abs()) <= 1.0
        assert of.sentinel_intact()
    if ob is not None:
        z = act_ref(y, act, act_param)
        lip = 1.1 if act == L.ACT_SILU else 1.0        # |d silu / dx| <= 1.1
        if ob.split_off:
            # hi + lo carries z to 2^-17 relative; the sm_90 SiLU (ex2 / rcp approximations) to ~2^-21
            assert excess(ob.value(), z, lip * sum_bound + 2.0 ** -16 * z.abs()) <= 1.0
        assert excess(ob.hi, z, lip * sum_bound + 2.0 ** -8 * z.abs()) <= 1.0   # round to nearest bf16: half an ulp
        assert ob.sentinel_intact()
    return y


def rand(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g) * scale


def linear_operands(g, cuda, rows, Cin, Ncols, *, ldb_pad=8):
    """x bf16 [rows, Cin] (NaN-padded view) and w bf16 [Ncols, Cin] (NaN-padded view: ldb > Ktot)."""
    x = poisoned(bf(rand(g, rows, Cin)).to(cuda))
    w = poisoned(bf(rand(g, Ncols, Cin, scale=Cin ** -0.5)).to(cuda), col_pad=ldb_pad, row_pad=0)
    return x, w


def row_view(x, NB, H, W):
    """Channels-last view of the [NB*H*W, C] operand x (x may be a slice of a wider buffer)."""
    ld = x.stride(0)
    return L.View(x, x.shape[1], W, H, NB, ld, W * ld, H * W * ld)


def k_groups_1x1(Cin, view=0):
    return [(view, 0, 0, 0, 0, (Cin + 63) // 64)]


# ---------------------------------------------------------------------------------------------------- tng_conv_gemm
@pytest.mark.parametrize("misaligned", [False, True])
@pytest.mark.parametrize("res_dt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("Ncols", [1, 2, 6, 36])
def test_gemm_scalar_epilogue(cuda, Ncols, res_dt, misaligned):
    """Ncols % 4 != 0 or a 16-byte-misaligned output (a column slice at +1 fp32 / +2 bf16 elements) takes the scalar
    epilogue (the vocoder's conv_post has Ncols = 1): bias, per-image vector, residual, alpha, activation, hi/lo with a gap
    between the halves. Cin = 72 with ldb = 80: the second K block overhangs both the view's C and Ktot."""
    g = torch.Generator().manual_seed(100 + Ncols)
    NB, H, W, Cin = 3, 1, 100, 72
    rows = NB * H * W
    x, w = linear_operands(g, cuda, rows, Cin, Ncols)
    bias = rand(g, Ncols).to(cuda)
    rowvec = poisoned_flat(rand(g, NB * Ncols).to(cuda), lead=1 if misaligned else 0)
    res = poisoned(rand(g, rows, Ncols).to(res_dt).to(cuda), col0=3 if misaligned else 0)
    act = L.ACT_SILU if Ncols % 2 else L.ACT_LRELU
    c0f, c0b = (1, 2) if misaligned else (0, 0)
    of = Out(rows, Ncols, dtype=torch.float32, device=cuda, col0=c0f, ld=c0f + Ncols + 12)
    ob = Out(rows, Ncols, dtype=torch.bfloat16, device=cuda, col0=c0b, split_off=Ncols + 5)
    check_gemm([row_view(x, NB, H, W)], k_groups_1x1(Cin), w, W, H, NB, of=of, ob=ob, act=act, act_param=0.2,
               bias=bias, rowvec=rowvec, res=res, alpha=0.75)


def test_gemm_every_n_tile_and_split_k(cuda):
    """One problem through every N tile (32, 64, 128, 160, 256) and the split-K plan the auto choice takes here (4 M
    tiles x 2 N tiles, 36 K blocks): each agrees with fp64 within the summation bound, and with the others."""
    g = torch.Generator().manual_seed(7)
    NB, H, W, Cin, Cout = 2, 16, 16, 256, 320
    rows = NB * H * W
    x = poisoned(bf(rand(g, rows, Cin)).to(cuda))
    wt = rand(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    pc = ops.PackedConv(wt, rand(g, Cout), split=False, device=cuda)
    views = ops.act_views(x, NB, H, W, Cin, False)
    groups = pc.groups()
    rowvec = rand(g, NB, Cout).to(cuda)
    res = poisoned(rand(g, rows, Cout).to(cuda))
    outs = {}
    for bn in (32, 64, 128, 160, 256, 0):
        kw = dict(bias=pc.bias, rowvec=rowvec, res=res, alpha=0.5, block_n=bn)
        of = Out(rows, Cout, dtype=torch.float32, device=cuda, ld=Cout + 12)
        fam = gemm_plan_family(views, groups, pc.weight, W, H, NB, out_f32=of.view, **kw)
        assert fam == (f"gemm_tc<{bn}>" if bn else "gemm_tc<160,splitk>")
        of = Out(rows, Cout, dtype=torch.float32, device=cuda, ld=Cout + 12)
        y = check_gemm(views, groups, pc.weight, W, H, NB, of=of, **kw)
        outs[bn] = of.hi.clone()
    _, absdot = gemm_reference(views, groups, pc.weight, W, H, NB, bias=pc.bias, rowvec=rowvec, res=res, alpha=0.5)
    for bn, o in outs.items():   # two results, each within the bound of fp64, are within twice the bound of each other
        assert excess(o, outs[128], 2 * GEMM_GAMMA * absdot.double() + 2 * U32 * y.double().abs()) <= 1.0


@pytest.mark.parametrize("NB,H,W,tail", [(16, 32, 2, "full tiles, 2 images per tile, bf16 only: no split-K"),
                                         (48, 2, 4, "full tiles, 16 images per tile: the per-slot image index"),
                                         (13, 2, 4, "ragged last tile of 5 images: the general epilogue"),
                                         (5, 4, 8, "ragged last tile of 1 image")])
def test_gemm_rowvec_several_images_per_tile(cuda, NB, H, W, tail):
    """The per-image row vector when one 128-row tile spans several images, with rowvec_ld > Ncols and the rowvec pointer
    offset into a wider NaN-padded buffer; a large per-image vector makes a wrong image index obvious."""
    g = torch.Generator().manual_seed(NB * 31 + H)
    Cin, Cout = 64, 64
    rows = NB * H * W
    x = poisoned(bf(rand(g, rows, Cin)).to(cuda))
    wt = rand(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    pc = ops.PackedConv(wt, rand(g, Cout), split=False, device=cuda)
    rv_ld = Cout + 12
    rvb = torch.full((NB + 1, rv_ld), NAN)
    rvb[:NB, :Cout] = rand(g, NB, Cout, scale=4.0)
    rowvec = poisoned_flat(rvb.reshape(-1).to(cuda), lead=4)        # 16-byte aligned: the vector epilogue
    ob = Out(rows, Cout, dtype=torch.bfloat16, device=cuda, ld=Cout + 24)
    check_gemm(ops.act_views(x, NB, H, W, Cin, False), pc.groups(), pc.weight, W, H, NB, ob=ob, bias=pc.bias,
               rowvec=rowvec, rowvec_ld=rv_ld)
    of = Out(rows, Cout, dtype=torch.float32, device=cuda, ld=Cout + 4)   # and with an fp32 output (split-K is off: K short)
    check_gemm(ops.act_views(x, NB, H, W, Cin, False), pc.groups(), pc.weight, W, H, NB, of=of, bias=pc.bias,
               rowvec=rowvec, rowvec_ld=rv_ld)


@pytest.mark.parametrize("rows", [512, 300])
def test_gemm_bf16_residual_with_ldr(cuda, rows):
    """res_dtype = BF16 with ldr > Ncols (NaN in the residual's padding), on full tiles and on a ragged last tile."""
    g = torch.Generator().manual_seed(rows)
    Cin, Ncols = 128, 192
    x, w = linear_operands(g, cuda, rows, Cin, Ncols)
    res = poisoned(bf(rand(g, rows, Ncols)).to(cuda), col_pad=24)
    of = Out(rows, Ncols, dtype=torch.float32, device=cuda, ld=Ncols + 16)
    ob = Out(rows, Ncols, dtype=torch.bfloat16, device=cuda, split_off=Ncols + 8)
    check_gemm([row_view(x, 1, 1, rows)], k_groups_1x1(Cin), w, rows, 1, 1, of=of, ob=ob, act=L.ACT_SILU,
               bias=rand(g, Ncols).to(cuda), res=res, alpha=0.5)


def skip_concat(g, cuda, NB, H, W, chans, a0s):
    """One view per source tensor: data channels [a0, a0 + C) of a NaN-padded buffer whose view starts `off` = 8 elements
    into each row (so s_w > C, a_c0 = a0 > 0, off > 0); channels [0, a0) of the view are NaN and must not be read."""
    rows = NB * H * W
    views, data = [], []
    for C, a0 in zip(chans, a0s):
        d = bf(rand(g, rows, C)).to(cuda)
        buf = poisoned(torch.full((rows, 8 + a0 + C), NAN, dtype=torch.bfloat16, device=cuda), col_pad=16)
        buf[:, 8 + a0:].copy_(d)
        ld = buf.stride(0)
        views.append(L.View(buf, a0 + C, W, H, NB, ld, W * ld, H * W * ld, off=8))
        data.append(d)
    return views, data


def skip_concat_groups(chans, a0s):
    """3x3 taps over the views of skip_concat, B packed as [Cout, tap * concat]: (k-groups, Ktot)."""
    Cs = sum(chans)
    groups, pre = [], [sum(chans[:i]) for i in range(len(chans))]
    for t in range(9):
        dh, dw = t // 3 - 1, t % 3 - 1
        for vi, (C, a0) in enumerate(zip(chans, a0s)):
            groups.append((vi, a0, dw, dh, t * Cs + pre[vi], (C + 63) // 64))
    return groups, 9 * Cs


@pytest.mark.parametrize("chans,a0s", [((72, 200), (16, 24)), ((64, 200, 72, 136), (8, 64, 40, 16))])
def test_gemm_multi_view_skip_concat(cuda, chans, a0s):
    """The skip-concat operand: 2-4 views with a_c0 > 0, s_w > C and off > 0, 3x3 taps, B packed densely over the
    concatenation with ldb > Ktot (NaN past Ktot). The last K block of each view overhangs its channels (72, 200) and,
    for the last view, Ktot: TMA must zero-fill both. Against the spec and against F.conv2d of the concatenation."""
    g = torch.Generator().manual_seed(sum(chans))
    NB, H, W, Cout = 2, 8, 16, 96
    views, data = skip_concat(g, cuda, NB, H, W, chans, a0s)
    Cs = sum(chans)
    wt = bf(rand(g, Cout, Cs, 3, 3, scale=(9 * Cs) ** -0.5))
    wk = wt.permute(0, 2, 3, 1).reshape(Cout, 9 * Cs)                     # [Cout, tap * concat]
    w = poisoned(wk.to(cuda), col_pad=8, row_pad=0)
    groups, _ = skip_concat_groups(chans, a0s)
    rows = NB * H * W
    of = Out(rows, Cout, dtype=torch.float32, device=cuda, ld=Cout + 8)
    ob = Out(rows, Cout, dtype=torch.bfloat16, device=cuda, split_off=Cout + 16)
    bias = rand(g, Cout)
    check_gemm(views, groups, w, W, H, NB, of=of, ob=ob, act=L.ACT_SILU, bias=bias.to(cuda))
    xc = torch.cat([d.float().cpu() for d in data], dim=1).view(NB, H, W, Cs).permute(0, 3, 1, 2).double()
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(rows, Cout)
    ref = nhwc(F.conv2d(xc, wt.double(), bias.double(), padding=1))
    absdot = nhwc(F.conv2d(xc.abs(), wt.double().abs(), bias.double().abs(), padding=1))
    assert excess(of.hi, ref, GEMM_GAMMA * absdot + U32 * ref.abs()) <= 1.0


@pytest.mark.parametrize("rows", [256, 200])
def test_gemm_accumulate_with_bf16_output(cuda, rows):
    """accumulate = True with an fp32 and a bf16 output: out_f32 += alpha * (acc + ...), and the bf16 output (with its
    activation and lo half) is derived from the ACCUMULATED value."""
    g = torch.Generator().manual_seed(rows + 1)
    Cin, Ncols = 64, 128
    x, w = linear_operands(g, cuda, rows, Cin, Ncols)
    prior = rand(g, rows, Ncols, scale=3.0).to(cuda)
    of = Out(rows, Ncols, dtype=torch.float32, device=cuda, ld=Ncols + 8, init=prior)
    ob = Out(rows, Ncols, dtype=torch.bfloat16, device=cuda, split_off=Ncols + 8)
    check_gemm([row_view(x, 1, 1, rows)], k_groups_1x1(Cin), w, rows, 1, 1, of=of, ob=ob, act=L.ACT_LRELU,
               act_param=0.1, prior=prior, bias=rand(g, Ncols).to(cuda), alpha=1.0 / 3)


@pytest.mark.parametrize("pad", [1, 0])
@pytest.mark.parametrize("split", [False, True])
def test_conv_stride2_odd_input(cuda, split, pad):
    """Stride 2 on odd H and W (parity views of unequal extents), padding 1, and the VAE encoder's pad (0, 1, 0, 1) +
    stride 2 + padding 0 (zero fill past the bottom / right edge), against F.conv2d in fp64."""
    g = torch.Generator().manual_seed(pad * 10 + split)
    NB, H, W, Cin, Cout = 2, 33, 15, 64, 96
    x = rand(g, NB, Cin, H, W)
    wt = rand(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5)
    b = rand(g, Cout)
    pc = ops.PackedConv(wt, b, split=split, device=cuda, stride=2, pad=pad)
    rows_in = x.permute(0, 2, 3, 1).reshape(-1, Cin)
    if split:
        hi = bf(rows_in)
        xin = torch.cat([hi, bf(rows_in - hi.float())], dim=1)
        xr, wr = x.double(), wt.double()
    else:
        xin = bf(rows_in)
        xr, wr = bf(x).double(), bf(wt).double()
    xin = poisoned(xin.to(cuda))
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    if pad == 0:    # zero padding on the bottom / right up to the last tap of the last output pixel
        xr = F.pad(xr, (0, 2 * Wo + 1 - W, 0, 2 * Ho + 1 - H))
    ref = F.conv2d(xr, wr, b.double(), stride=2, padding=pad)
    absdot = F.conv2d(xr.abs(), wr.abs(), b.double().abs(), stride=2, padding=pad)
    assert ref.shape[-2:] == (Ho, Wo)
    of = Out(NB * Ho * Wo, Cout, dtype=torch.float32, device=cuda, ld=Cout + 4)
    ops.run_conv(pc, xin, NB, H, W, out_f32=of.view)
    torch.cuda.synchronize()
    nhwc = lambda t: t.permute(0, 2, 3, 1).reshape(-1, Cout)
    # split operands drop the lo*lo product (<= 2^-16 |ab| each) on top of the fp32 summation
    gam = 2 * GEMM_GAMMA if split else GEMM_GAMMA
    assert excess(of.hi, nhwc(ref), gam * nhwc(absdot)) <= 1.0
    assert of.sentinel_intact()


@pytest.mark.parametrize("case", ["fused epilogue, ld_f32 > Ncols", "after-pass: ragged tiles", "after-pass: accumulate",
                                  "after-pass: split-K"])
def test_gemm_groupnorm_statistics_every_variant(cuda, case):
    """gn_stats on each way the statistics are produced; they must equal the per-(image, channel) column sums of what was
    stored: fp32 partials over <= 128 rows, so |error| <= 128 * 2^-24 * sum |x| (and sum x^2)."""
    g = torch.Generator().manual_seed(len(case))
    NB, H, W, Cin, Cout = (4, 8, 16, 64, 128) if "fused" in case or "accumulate" in case else \
        (3, 12, 16, 64, 96) if "ragged" in case else (2, 16, 16, 256, 320)
    rows = NB * H * W
    x = poisoned(bf(rand(g, rows, Cin)).to(cuda))
    pc = ops.PackedConv(rand(g, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5), rand(g, Cout) + 2.0, split=False, device=cuda)
    views = ops.act_views(x, NB, H, W, Cin, False)
    acc = "accumulate" in case
    prior = rand(g, rows, Cout).to(cuda) if acc else None
    of = Out(rows, Cout, dtype=torch.float32, device=cuda, ld=Cout + 12, init=prior)
    st = torch.zeros(NB, Cout, 2, dtype=torch.float64, device=cuda)
    kw = dict(bias=pc.bias, gn_stats=st, stats_hw=H * W, accumulate=acc)
    fam = gemm_plan_family(views, pc.groups(), pc.weight, W, H, NB,
                           out_f32=Out(rows, Cout, dtype=torch.float32, device=cuda, ld=Cout + 12, init=prior).view, **kw)
    assert ("splitk" in fam) == ("split-K" in case)
    st.zero_()
    check_gemm(views, pc.groups(), pc.weight, W, H, NB, of=of, prior=prior, **kw)
    o = of.hi.double().cpu().view(NB, H * W, Cout)
    bound = 128 * U32
    assert excess(st[..., 0], o.sum(1), bound * o.abs().sum(1)) <= 1.0
    assert excess(st[..., 1], (o * o).sum(1), bound * (o * o).sum(1)) <= 1.0


# ---------------------------------------------------------------------------------------------------- GEGLU epilogue
GELU_LIP = 1.13   # max |d gelu / dx| of both forms (1.129 at x ~ 1.41)


def gelu64(x, tanh):
    """fp64 GELU. The erf form through erfc and the tanh form as x * sigmoid(2u): neither cancels in the negative tail,
    where 0.5 x (1 + tanh u) loses every digit (a 58 % "error" at x ~ -10)."""
    x = x.double()
    if tanh:
        return x * torch.sigmoid(2.0 * math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3))
    return 0.5 * x * torch.erfc(-x / math.sqrt(2.0))


def geglu_halves(t, bn):
    """[rows, Ncols] in the per-N-tile layout (BN/2 hidden columns, then their BN/2 gate columns) -> (hidden, gate),
    each [rows, Ncols / 2] in output column order (tile tn at columns tn * BN/2)."""
    v = t.double().reshape(t.shape[0], -1, bn)
    return v[..., :bn // 2].reshape(t.shape[0], -1), v[..., bn // 2:].reshape(t.shape[0], -1)


def geglu_reference(y, absdot, bn, tanh, *, gamma=GEMM_GAMMA):
    """z = hidden * gelu(gate) in fp64 and its per-element allowance before the output rounding: gamma S_h |gelu(g)|
    (summation error of the hidden half) + 1.13 |h| gamma S_g (of the gate half, through |gelu'| <= 1.13) + |h| |g| 2^-21
    (the kernel's GELU: its formula is within 1.8e-7 |x| of the exact one, the ex2 / rcp approximations add <= 2^-22 |x|;
    an absolute term, since the erf form's relative error reaches 1.6e-3 at x = -5). S_h / S_g: |operand| contractions."""
    h, gt = geglu_halves(y, bn)
    sh, sg = geglu_halves(absdot, bn)
    gg = gelu64(gt, tanh)
    return h * gg, gamma * sh * gg.abs() + GELU_LIP * h.abs() * gamma * sg + h.abs() * gt.abs() * 2.0 ** -21


def geglu_weights(g, Ncols, bn, Cin):
    """fp32 weight [Ncols, Cin] and bias for BN-column tiles whose second half is the gate: gate rows are halved and the
    gate bias spreads over [-8.5, 8.5] in every tile, so the gates cover about [-9, 9] (both GELU tails); the hidden bias
    is 1 + N(0, 0.5^2), so swapped halves cannot pass."""
    gate = (torch.arange(Ncols) % bn) >= bn // 2
    w = rand(g, Ncols, Cin, scale=Cin ** -0.5)
    w[gate] *= 0.5
    bias = 1.0 + 0.5 * rand(g, Ncols)
    bias[gate] = torch.linspace(-8.5, 8.5, Ncols // 2)[torch.randperm(Ncols // 2, generator=g)]
    return w, bias


def geglu_operands(g, device, rows, bn, *, Cin=72):
    """Two N tiles of a GEGLU GEMM: x bf16 [rows, Cin] (NaN-padded view), w bf16 [2 BN, Cin] in the kernel's per-tile
    layout (NaN-padded view, ldb = 80 > Ktot = 72: the K block overhangs both), fp32 bias."""
    w, bias = geglu_weights(g, 2 * bn, bn, Cin)
    x = poisoned(bf(rand(g, rows, Cin)).to(device))
    return x, poisoned(bf(w).to(device), col_pad=8, row_pad=0), bias.to(device)


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("rows", [256, 300])
@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("tanh", [False, True])
def test_geglu_epilogue_every_instantiation(cuda, tanh, bn, rows, split):
    """Every epi_tile_geglu instantiation: {erf, tanh} x BN {128, 256} x {full tiles (256 rows), a ragged last tile (300
    rows: 44 live)} x {bf16, hi/lo}, over two N tiles so that the second writes at output column BN/2. The output sits at
    column 8 of a wider buffer (ld_bf16 > width, a gap before the lo half); everything around it keeps its sentinel."""
    g = torch.Generator().manual_seed(bn + rows + 2 * split + 4 * tanh)
    x, w, bias = geglu_operands(g, cuda, rows, bn)
    views, groups = [row_view(x, 1, 1, rows)], k_groups_1x1(x.shape[1])
    ob = Out(rows, bn, dtype=torch.bfloat16, device=cuda, col0=8, split_off=bn + 8 if split else 0, ld=2 * bn + 32)
    L.conv_gemm(views, groups, w, rows, 1, 1, bias=bias, out_bf16=ob.view, act=L.ACT_GEGLU_TANH if tanh else L.ACT_GEGLU,
                split_off=ob.split_off, block_n=bn)
    torch.cuda.synchronize()
    y, absdot = gemm_reference(views, groups, w, rows, 1, 1, bias=bias)
    gate = geglu_halves(y, bn)[1]
    assert gate.min() < -8 and gate.max() > 8
    z, bound = geglu_reference(y, absdot, bn, tanh)
    e = excess(ob.hi, z, bound + 2.0 ** -8 * z.abs())       # round to nearest bf16: half an ulp <= 2^-8 |z|
    if split:                                                 # hi + lo carries z to 2^-17
        e = max(e, excess(ob.value(), z, bound + 2.0 ** -16 * z.abs()))
    print(f"geglu {'tanh' if tanh else 'erf'} BN={bn} rows={rows} {'hi/lo' if split else 'bf16'}: worst excess {e:.3f}")
    assert e <= 1.0
    assert ob.sentinel_intact()


def geglu_linear_reference(x, wt, b, tanh, *, gamma):
    """fp64 F.linear(x, wt, b).chunk(2) -> hidden * gelu(gate) (the diffusers / T5 GEGLU) with the geglu_reference
    allowance: the whole output is one 'tile' of BN = Ncols."""
    y = F.linear(x.double(), wt.double(), b.double())
    absdot = F.linear(x.double().abs(), wt.double().abs(), b.double().abs())
    return geglu_reference(y, absdot, wt.shape[0], tanh, gamma=gamma)


@pytest.mark.parametrize("tanh", [False, True])
def test_geglu_packed_conv_split(cuda, tanh):
    """ops.PackedConv(geglu_bn=256) in split mode, as the UNet feed-forward (and T5 with the tanh form) packs it: the host
    interleave of the hidden / gate rows and of the bias, hi/lo weights and operand, through tng_conv_gemm, against fp64
    F.linear + hidden * gelu(gate) of the fp32 weights; 200 rows (ragged), inner = 256 (two N tiles). The 3-term split
    products drop lo * lo (<= 2^-16 |x w| each with the lo rounding): gamma = 2 Gamma, as for the split convolutions."""
    g = torch.Generator().manual_seed(11 + tanh)
    rows, Cin, inner = 200, 128, 256
    x = rand(g, rows, Cin)
    wt, b = geglu_weights(g, 2 * inner, 2 * inner, Cin)
    pc = ops.PackedConv(wt, b, split=True, device=cuda, geglu_bn=256, geglu_tanh=tanh)
    xin = poisoned(torch.cat(pack_split(x), dim=1).to(cuda))
    ob = Out(rows, inner, dtype=torch.bfloat16, device=cuda, split_off=inner, ld=2 * inner)
    ops.run_linear(pc, xin, out_bf16=ob.view)
    torch.cuda.synchronize()
    z, bound = geglu_linear_reference(x, wt, b, tanh, gamma=2 * GEMM_GAMMA)
    e = excess(ob.value(), z, bound + 2.0 ** -16 * z.abs())
    print(f"geglu PackedConv split {'tanh' if tanh else 'erf'}: worst excess {e:.3f}")
    assert e <= 1.0
    assert ob.sentinel_intact()


# ---------------------------------------------------------------------------------------------------- tng_attention
def attn_ref(q, k, v, *, batch, heads, Lq, Lk, scale, kbias=None, width=64):
    """fp64 softmax(q k^T * scale + kbias) v and softmax |v| (the per-element scale of the P rounding error);
    q / k / v: [rows, heads * width] fp64."""
    qh = q.view(batch, Lq, heads, width).transpose(1, 2)
    kh = k.view(batch, Lk, heads, width).transpose(1, 2)
    vh = v.view(batch, Lk, heads, width).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) * scale
    if kbias is not None:
        s = s + kbias.double().view(batch, 1, 1, Lk)
    p = s.softmax(-1)
    back = lambda t: t.transpose(1, 2).reshape(batch * Lq, heads * width)
    return back(p @ vh), back(p @ vh.abs())


def attn_operands(g, B, heads, L_, *, offset_dim=None):
    C = heads * 64
    t = rand(g, B * L_, C, scale=0.7)
    if offset_dim is not None:   # a shared component along one head dimension: q . k ~ -32 (score ~ -4 at scale 1/8)
        t.view(B * L_, heads, 64)[:, :, 0] = offset_dim
    return t


def pack_split(t):
    hi = bf(t)
    return hi, bf(t - hi.float())


def fused_buffer(parts, cuda, *, lead=8, gap=8, tail=24):
    """Columns [lead NaN | part0 | gap NaN | part1 | part2 ... | tail NaN] of one row-major bf16 buffer (+ NaN rows):
    returns (buffer view, first column of every part)."""
    rows = parts[0].shape[0]
    cols, c = [], lead
    for i, p in enumerate(parts):
        cols.append(c)
        c += p.shape[1] + (gap if i == 0 else 0)
    ld = c + tail
    ld += (-ld) % 8
    buf = torch.full((rows + 5, ld), NAN, dtype=torch.bfloat16, device=cuda)
    for p, c0 in zip(parts, cols):
        buf[:rows, c0:c0 + p.shape[1]] = p.to(cuda)
    return buf[:rows], cols


def run_attention_case(cuda, B, heads, Lq, Lk, nsplit, kbias=None, seed=0, offset=True):
    g = torch.Generator().manual_seed(seed)
    C = heads * 64
    q = attn_operands(g, B, heads, Lq, offset_dim=4.0 if offset else None)
    k = attn_operands(g, B, heads, Lk, offset_dim=-8.0 if offset else None)
    v = attn_operands(g, B, heads, Lk) + 0.5
    if nsplit == 1:
        qb, kb_, vb = bf(q), bf(k), bf(v)
        qbuf, (qc,) = fused_buffer([qb], cuda)
        kvbuf, (kc, vc) = fused_buffer([kb_, vb], cuda)
        lo = dict()
        qr, kr, vr = qb.double(), kb_.double(), vb.double()
    else:
        (qh, ql), (kh, kl), (vh, vl) = pack_split(q), pack_split(k), pack_split(v)
        qbuf, (qc, _) = fused_buffer([qh, ql], cuda, gap=0)
        kvbuf, (kc, _, vc, _) = fused_buffer([kh, kl, vh, vl], cuda, gap=0)
        lo = dict(q_lo_off=C, k_lo_off=C, v_lo_off=C)
        qr, kr, vr = (h.double() + l_.double() for h, l_ in ((qh, ql), (kh, kl), (vh, vl)))
    split_off = C + 8
    out = Out(B * Lq, C, dtype=torch.bfloat16, device=cuda, split_off=split_off, ld=2 * C + 24)
    kb_dev = None if kbias is None else poisoned_flat(kbias.to(cuda))
    L.attention(qbuf, kvbuf, kvbuf, out.view, batch=B, heads=heads, Lq=Lq, Lk=Lk, scale=0.125, q_col0=qc, k_col0=kc,
                v_col0=vc, kbias=kb_dev, nsplit=nsplit, split_off=split_off, **lo)
    torch.cuda.synchronize()
    ref, pv = attn_ref(qr, kr, vr, batch=B, heads=heads, Lq=Lq, Lk=Lk, scale=0.125, kbias=kbias)
    assert out.sentinel_intact()
    if nsplit == 1:
        # P enters the PV product rounded to bf16 (<= 2^-8 relative each, the normaliser keeps the fp32 values) and the
        # output is rounded to bf16: |err| <= 2^-8 sum p |v| + 2^-8 |o|, with a 2x margin on the first term
        assert excess(out.hi, ref, 2.0 ** -7 * pv + 2.0 ** -8 * ref.abs()) <= 1.0
        assert excess(out.value(), ref, 2.0 ** -7 * pv + 2.0 ** -15 * ref.abs()) <= 1.0
    else:
        # 3-term split products: the dropped lo*lo terms (~2^-16 relative) of the scores (|q.k| * scale <= ~8 here) and
        # of PV, plus the lo half rounding; 2^-11 sum p |v| covers the score error e^(8 * 2^-16) - 1 ~ 2^-13 with margin
        assert excess(out.value(), ref, 2.0 ** -11 * pv + 2.0 ** -15 * ref.abs()) <= 1.0
        assert rowcol_err(out.value(), ref) < 2e-3
    return out, ref


@pytest.mark.parametrize("B,heads,Lq,Lk", [(2, 2, 127, 1), (2, 2, 129, 7), (1, 3, 1, 63), (2, 2, 127, 64),
                                           (2, 2, 129, 65), (1, 2, 1, 129), (1, 20, 129, 77), (2, 20, 64, 129)])
@pytest.mark.parametrize("nsplit", [1, 2])
def test_attention_sequence_edges_sliced_operands(cuda, B, heads, Lq, Lk, nsplit):
    """Ragged key tiles (Lk = 1, 7, 63, 64, 65 = one live key in the last tile, 129), Lq = 1 / 127 / 129, heads = 20,
    q / k / v at non-zero columns of fused NaN-padded buffers, hi/lo output with a gap and ld_o > width. Scores are
    biased to ~ -4 so that a key past Lk (score 0 from the zero-filled tile) would dominate the row."""
    run_attention_case(cuda, B, heads, Lq, Lk, nsplit, seed=Lq * 1000 + Lk + heads)


@pytest.mark.parametrize("mask", ["one 64-key tile", "all keys but one", "all keys"])
def test_attention_masking(cuda, mask):
    """kbias of -10000 over a whole 64-key tile, over all keys but one, and over every key (all scores shift alike:
    the plain softmax of the unmasked scores, as torch gives)."""
    B, heads, Lq, Lk = 2, 2, 100, 200
    kb = torch.zeros(B, Lk)
    if mask == "one 64-key tile":
        kb[:, 64:128] = -10000.0
    elif mask == "all keys but one":
        kb[:, :] = -10000.0
        kb[0, 150] = 0.0
        kb[1, 3] = 0.0
    else:
        kb[:, :] = -10000.0
    out, ref = run_attention_case(cuda, B, heads, Lq, Lk, 1, kbias=kb, seed=len(mask), offset=False)
    if mask == "all keys but one":   # the output rows are that key's value row (rounded to bf16)
        assert torch.equal(out.hi.cpu().view(B, Lq, -1)[0], bf(ref.view(B, Lq, -1)[0]).expand(Lq, -1))


@pytest.mark.parametrize("L_,spread", [(128, 1.0), (384, 1.0), (384, 6.0)])
def test_attention_wide_sliced_operands(cuda, L_, spread):
    """tng_attention_wide (the VAE AttnBlock: one head of width 512) with B = 2, q / k / v at non-zero columns of one
    NaN-padded fused buffer (ld > 3 * 512) and an output at a column offset with ld_o > 512: both 256-column halves land
    in place and the padding stays untouched. `spread` > 1 makes the key magnitudes grow along the sequence so that the
    running row maximum moves. Same per-element bound as the bf16 head-64 kernel."""
    B, C = 2, 512
    g = torch.Generator().manual_seed(L_ + int(spread))
    q = bf(rand(g, B * L_, C))
    k = bf(rand(g, B * L_, C) * torch.linspace(1.0, spread, L_).repeat(B)[:, None])
    v = bf(rand(g, B * L_, C) + 0.5)
    buf, (qc, kc, vc) = fused_buffer([q, k, v], cuda)
    assert buf.stride(0) > 3 * C and min(qc, kc, vc) > 0
    out = Out(B * L_, C, dtype=torch.bfloat16, device=cuda, col0=8, ld=C + 24)
    L.attention_wide(buf, buf, buf, out.view, batch=B, L=L_, dim=C, scale=C ** -0.5, q_col0=qc, k_col0=kc, v_col0=vc)
    torch.cuda.synchronize()
    ref, pv = attn_ref(q.double(), k.double(), v.double(), batch=B, heads=1, Lq=L_, Lk=L_, scale=C ** -0.5, width=C)
    assert out.sentinel_intact()
    assert excess(out.hi, ref, 2.0 ** -7 * pv + 2.0 ** -8 * ref.abs()) <= 1.0


# ---------------------------------------------------------------------------------------------------- tng_sched_step
def coef_rows():
    """Coefficient rows from the product's own scheduler tables: (name, row, uses clip)."""
    rows = []
    for name, sch in (("ddpm-eps-clip", DDPMScheduler(beta_schedule="scaled_linear", beta_start=0.00085,
                                                      beta_end=0.012, prediction_type="epsilon", clip_sample=True)),
                      ("ddpm-v", DDPMScheduler(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012,
                                               prediction_type="v_prediction", clip_sample=False)),
                      ("ddim-eps", DDIMScheduler(prediction_type="epsilon", clip_sample=False)),
                      ("ddim-v", DDIMScheduler(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012,
                                               prediction_type="v_prediction", clip_sample=False))):
        sch.set_timesteps(50)
        tab = sch.coefficient_table()
        rows.append((name, tab[20].clone()))
    return rows


@pytest.mark.parametrize("layout", ["cfg, noise, hi/lo next_in, prev aliases sample",
                                    "no cfg, no noise, plain next_in, separate prev",
                                    "cfg, noise, prev only",
                                    "no cfg, noise, hi/lo next_in only",
                                    "initial packing (model_out NULL)"])
@pytest.mark.parametrize("row", range(4))
def test_sched_step_bit_exact(cuda, row, layout):
    """tng_sched_step equals spec_sched_step bit for bit on coefficient rows of DDPM / DDIM, epsilon / v prediction
    and x0 clipping; model_out with ld_mo > C, next_in with ld_in > C (hi/lo with a gap), prev aliasing sample, and
    B * C * HW = 888, not a multiple of the 256-thread block."""
    name, coef = coef_rows()[row]
    assert (float(coef[8]) > 0) == ("clip" in name)
    B, Cc, HW = 3, 8, 37
    cfg = layout.startswith("cfg")
    g = torch.Generator().manual_seed(row * 10 + len(layout))
    n_mo = (2 if cfg else 1) * B * HW
    mo = None if "NULL" in layout else poisoned(rand(g, n_mo, Cc, scale=1.5).to(cuda), col_pad=8, align=4)
    sample = rand(g, B, Cc, HW, scale=1.3).to(cuda)
    noise = rand(g, B, Cc, HW).to(cuda) if "noise" in layout and "no noise" not in layout else None
    if "NULL" in layout:
        noise = None
    split = "hi/lo" in layout or "NULL" in layout
    has_next = "next_in" in layout or "NULL" in layout
    nin = Out((2 if cfg else 1) * B * HW, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 8 if split else 0,
              ld=2 * Cc + 16) if has_next else None
    alias = "aliases" in layout
    prev = None if "only" in layout and "prev only" not in layout else \
        (sample if alias else torch.full((B, Cc, HW), NAN, device=cuda))
    coef_d = poisoned_flat(coef.to(cuda), lead=4)
    # the spec on CPU copies (same aliasing)
    s_c = sample.cpu().clone()
    p_c = None if prev is None else (s_c if alias else prev.cpu().clone())
    n_c = None if nin is None else nin.cpu_clone()
    S.spec_sched_step(None if mo is None else mo.cpu(), cfg, 3.0, s_c, None if noise is None else noise.cpu(), coef,
                      p_c, None if n_c is None else n_c.view, B=B, Cc=Cc, HW=HW,
                      split_off=0 if nin is None else nin.split_off)
    L.sched_step(mo, cfg, 3.0, sample, noise, coef_d, prev, None if nin is None else nin.view, B=B, Cc=Cc, HW=HW,
                 split_off=0 if nin is None else nin.split_off)
    torch.cuda.synchronize()
    if prev is not None:
        assert torch.equal(prev.cpu(), p_c)
    if nin is not None:
        assert torch.equal(nin.buf.cpu(), n_c.buf)    # every element, the sentinels included
    if "clip" in name and mo is not None:             # the clip row actually clips here
        c = coef.tolist()
        v = mo.cpu()[:B * HW].view(B, HW, Cc).transpose(1, 2) if not cfg else None
        if v is not None:
            x0 = (c[0] * sample.cpu() + c[1] * v) / c[9]
            assert (x0.abs() > c[8]).any()


# ---------------------------------------------------------------------------------------------------- tng_dpm_step
def dpm_rows():
    """(name, order, row) from the product's own tables: the order 1, 2 and 3 rows (steps 0, 1 and 5 of a 20-step grid)
    of a solver_order = 3 DPM-Solver++ and DPM-Solver, epsilon and v prediction."""
    rows = []
    for algo in ("dpmsolver++", "dpmsolver"):
        for pred in ("epsilon", "v_prediction"):
            s = DPMSolverMultistepScheduler(beta_schedule="scaled_linear", beta_start=0.00085, beta_end=0.012,
                                            prediction_type=pred, algorithm_type=algo, solver_order=3)
            s.set_timesteps(20)
            tab = s.coefficient_table()
            for i in (0, 1, 5):
                rows.append((f"{algo}-{pred}", s.order_at(i), tab[i].clone()))
    return rows


@pytest.mark.parametrize("layout", ["cfg, hi/lo next_in, prev aliases sample",
                                    "no cfg, plain next_in, separate prev",
                                    "cfg, prev only",
                                    "no cfg, hi/lo next_in only"])
@pytest.mark.parametrize("row", range(12))
def test_dpm_step_bit_exact(cuda, row, layout):
    """tng_dpm_step equals spec_dpm_step bit for bit on order 1 / 2 / 3 rows of DPM-Solver(++) with epsilon and v
    prediction: CFG or not, model_out with ld_mo > C (NaN padding), prev aliasing sample / separate / NULL, next_in plain
    or hi/lo with a gap (compared over the whole buffer, sentinels included), history slots m1 / m2 NaN-padded past
    B * C * HW = 888 (not a multiple of the 256-thread block), and m0 followed by a sentinel tail."""
    name, order, coef = dpm_rows()[row]
    B, Cc, HW = 3, 8, 37
    n = B * Cc * HW
    cfg = layout.startswith("cfg")
    g = torch.Generator().manual_seed(row * 10 + len(layout))
    mo = poisoned(rand(g, (2 if cfg else 1) * B * HW, Cc, scale=1.5).to(cuda), col_pad=8, align=4)
    sample = rand(g, B, Cc, HW, scale=1.3).to(cuda)
    m1 = poisoned_flat(rand(g, n).to(cuda)) if order >= 2 else None
    m2 = poisoned_flat(rand(g, n).to(cuda)) if order == 3 else None
    m0 = Out(1, n, dtype=torch.float32, device=cuda, ld=n, row_pad=1)
    split = "hi/lo" in layout
    nin = Out((2 if cfg else 1) * B * HW, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 8 if split else 0,
              ld=2 * Cc + 16) if "next_in" in layout else None
    alias = "aliases" in layout
    prev = None if "next_in only" in layout else (sample if alias else torch.full((B, Cc, HW), NAN, device=cuda))
    # the spec on CPU copies (same aliasing)
    s_c = sample.cpu().clone()
    p_c = None if prev is None else (s_c if alias else prev.cpu().clone())
    m0_c = m0.cpu_clone()
    n_c = None if nin is None else nin.cpu_clone()
    S.spec_dpm_step(mo.cpu(), cfg, 3.0, s_c, coef, order, m0_c.buf[0], None if m1 is None else m1.cpu(),
                    None if m2 is None else m2.cpu(), p_c, None if n_c is None else n_c.view, B=B, Cc=Cc, HW=HW,
                    split_off=0 if nin is None else nin.split_off)
    L.dpm_step(mo, cfg, 3.0, sample, poisoned_flat(coef.to(cuda), lead=4), order, m0.buf[0], m1, m2, prev,
               None if nin is None else nin.view, B=B, Cc=Cc, HW=HW, split_off=0 if nin is None else nin.split_off)
    torch.cuda.synchronize()
    assert torch.equal(m0.buf.cpu(), m0_c.buf), name    # every element, the sentinel tail included
    if prev is not None:
        assert torch.equal(prev.cpu(), p_c), name
    if nin is not None:
        assert torch.equal(nin.buf.cpu(), n_c.buf), name


# ---------------------------------------------------------------------------------------------------- GroupNorm
def group_fit(got, ref, NB, HW, groups):
    """Per (image, group) least-squares fit got ~ a * ref + b (gamma = 1, beta = 0, so ref is the normalised value):
    a - 1 is the relative rstd error, b the mean error in units of the group's std. Returns (max |a - 1|, max |b|,
    max residual)."""
    got, ref = got.double().cpu(), ref.double().cpu()
    C_ = ref.shape[1]
    gv = lambda t: t.view(NB, HW, groups, C_ // groups).permute(0, 2, 1, 3).reshape(NB, groups, -1)
    x, y = gv(ref), gv(got)
    xm, ym = x.mean(-1, keepdim=True), y.mean(-1, keepdim=True)
    a = ((x - xm) * (y - ym)).sum(-1) / (x - xm).pow(2).sum(-1)
    b = ym.squeeze(-1) - a * xm.squeeze(-1)
    resid = (y - (a[..., None] * x + b[..., None])).abs().max()
    return (a - 1).abs().max().item(), b.abs().max().item(), resid.item()


# |mean| / std -> bound on the relative rstd error and on the mean error (in stds) of split mode. The ratio-100 bound
# is ~3x the rstd error measured on an H100 80GB HBM3 (700 W power limit): 1.7e-5 (mean error 6.8e-6 std)
GN_ENVELOPE = {1: 2e-5, 10: 2e-5, 30: 2e-5, 100: 5e-5}


@pytest.mark.parametrize("ratio", [1, 10, 30, 100])
def test_groupnorm_accuracy_envelope(cuda, ratio):
    """Stand-alone statistics + apply in split mode on off-centre inputs, against fp64 F.group_norm.
    Where the error comes from: the per-channel sums S, Q are fp32 partials over <= 128 rows (fp64 across partials),
    and var = Q/n - mean^2 cancels: Q/n ~ mean^2 (1 + (std/mean)^2), so the fp32 relative error of Q (~2^-24 * a few)
    grows by (mean/std)^2 in var, i.e. rstd error ~ 2^-24 * r^2. A CPU emulation with 43-row partials predicts
    5e-7 / 7e-6 / 7e-5 at r = 10 / 30 / 100; measured on an H100 (16-row partials at this shape): 1.8e-7 / 9.8e-7 /
    1.7e-5. The split-mode bound of 2e-5 holds through r = 30; fp32 group sums instead of fp64 break it at r = 30."""
    g = torch.Generator().manual_seed(ratio)
    NB, HW, Cc, groups = 2, 4096, 320, 32
    std = 0.5
    sign = torch.where((torch.arange(Cc) // (Cc // groups)) % 2 == 0, 1.0, -1.0)   # per group: +-ratio * std
    x = (rand(g, NB * HW, Cc) * std + ratio * std * sign[None]).to(cuda)
    st = torch.zeros(NB, Cc, 2, dtype=torch.float64, device=cuda)
    L.groupnorm_stats(x, NB, HW, st)
    y = Out(NB * HW, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc, ld=2 * Cc + 8)
    ones, zeros = torch.ones(Cc, device=cuda), torch.zeros(Cc, device=cuda)
    L.groupnorm(x, st, None, None, NB, HW, groups, ones, zeros, 1e-5, L.ACT_NONE, y.view, split_off=Cc)
    torch.cuda.synchronize()
    ref = F.group_norm(x.double().cpu().view(NB, HW, Cc).permute(0, 2, 1), groups, eps=1e-5)
    ref = ref.permute(0, 2, 1).reshape(NB * HW, Cc)
    da, db, resid = group_fit(y.value(), ref, NB, HW, groups)
    print(f"groupnorm |mean|/std={ratio}: rstd rel err {da:.2e}, mean err {db:.2e} std, residual {resid:.2e}")
    assert da <= GN_ENVELOPE[ratio] and db <= GN_ENVELOPE[ratio]
    # what is left after the per-group affine error: the fp32 fma x * sc + sh with |x * sc| ~ r (ulp(r) ~ r * 2^-23)
    # and the rounding of the lo half (hi + lo carries a value to 2^-17 relative)
    assert resid <= ratio * 2.0 ** -21 + 2.0 ** -16 * ref.abs().max().item()
    assert y.sentinel_intact()


@pytest.mark.parametrize("C0,C1,groups,HW,dt1", [(1280, 1280, 32, 37, torch.bfloat16), (1280, 640, 32, 4, torch.float32),
                                                  (96, 0, 32, 37, None), (96, 64, 32, 4, torch.bfloat16),
                                                  (320, 0, 32, 1, None), (640, 320, 32, 37, torch.float32)])
def test_groupnorm_shapes(cuda, C0, C1, groups, HW, dt1):
    """Wide concatenations (several channel slabs), C / groups = 3 (not a multiple of 4), groups straddling the concat
    boundary (96 + 64 channels in groups of 5), HW = 1 / 4 / 37, a bf16 x1; the stand-alone statistics pass reads a
    bf16 input through ld > C. Statistics: fp32 partials over <= 128 rows -> |err| <= 128 * 2^-24 * sum |x|."""
    NB = 3
    g = torch.Generator().manual_seed(C0 + C1 + HW)
    Cc = C0 + C1
    x0 = (rand(g, NB * HW, C0) * 2 + 0.5).to(cuda)
    x1 = (rand(g, NB * HW, C1) - 0.3).to(dt1).to(cuda) if C1 else None
    gamma, beta = rand(g, Cc).to(cuda), rand(g, Cc).to(cuda)
    st0 = torch.zeros(NB, C0, 2, dtype=torch.float64, device=cuda)
    st1 = torch.zeros(NB, C1, 2, dtype=torch.float64, device=cuda) if C1 else None
    L.groupnorm_stats(poisoned(x0, col_pad=12, align=4), NB, HW, st0)
    if C1:
        L.groupnorm_stats(poisoned(x1, col_pad=16), NB, HW, st1)
    for x, st in ((x0, st0), (x1, st1)):
        if x is None:
            continue
        xd = x.double().cpu().view(NB, HW, -1)
        assert excess(st[..., 0], xd.sum(1), 128 * U32 * xd.abs().sum(1)) <= 1.0
        assert excess(st[..., 1], (xd * xd).sum(1), 128 * U32 * (xd * xd).sum(1)) <= 1.0
    y = Out(NB * HW, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 8, ld=2 * Cc + 24)
    raw = Out(NB * HW, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 16, ld=2 * Cc + 32)
    L.groupnorm(x0, st0, x1, st1, NB, HW, groups, gamma, beta, 1e-5, L.ACT_SILU, y.view, split_off=y.split_off,
                raw=raw.view, raw_split_off=raw.split_off)
    torch.cuda.synchronize()
    xc = x0.double() if x1 is None else torch.cat([x0.double(), x1.double()], dim=1)
    xc = xc.cpu()
    ref = F.group_norm(xc.view(NB, HW, Cc).permute(0, 2, 1), groups, gamma.double().cpu(), beta.double().cpu(), 1e-5)
    ref = F.silu(ref).permute(0, 2, 1).reshape(NB * HW, Cc)
    # hi + lo carries a value to 2^-17 relative (the lo half is rounded too); the fp32 apply and the SiLU
    # approximations add ~2^-21 of the values
    rms = ref.pow(2).mean().sqrt().item()
    assert excess(y.value(), ref, 2.0 ** -16 * ref.abs() + 2.0 ** -18 * rms) <= 1.0
    assert rowcol_err(y.value(), ref) < 2e-4
    assert el_err(y.hi, ref) < 2.0 ** -8 * (ref.abs().max() / ref.pow(2).mean().sqrt()).item() * 1.01
    assert excess(raw.value(), xc, 2.0 ** -16 * xc.abs() + 1e-30) <= 1.0   # hi + lo holds fp32 to 2^-17
    assert y.sentinel_intact() and raw.sentinel_intact()


# ---------------------------------------------------------------------------------------------------- LayerNorm / RMSNorm
@pytest.mark.parametrize("Cc", [4, 128, 132, 256, 260, 640, 1280, 2048])
def test_layernorm_rmsnorm_template_boundaries(cuda, Cc):
    """LayerNorm and RMSNorm at the boundaries of the row-cache template (NI = ceil(C / 128)), with ld_y > 2C (hi/lo with
    a gap) and inputs centred at 1000 (std 1): against fp64."""
    rows = 67
    g = torch.Generator().manual_seed(Cc)
    x = (rand(g, rows, Cc) + 1000.0).to(cuda)
    gamma, beta = rand(g, Cc).to(cuda), rand(g, Cc).to(cuda)
    ni = (Cc // 4 + 31) // 32
    xd = x.double().cpu()
    # hi + lo carries a value to 2^-17 relative. The mean is an fp32 sum: each lane adds 2 NI pairs in sequence, then 5 butterfly steps, so
    # |d mean| <= (2 NI + 6) 2^-24 mean|x|, which moves every normalised value by d mean * rstd * |gamma|
    y = Out(rows, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 4, ld=2 * Cc + 12)
    L.layernorm(x, gamma, beta, 1e-5, y.view, split_off=y.split_off)
    torch.cuda.synchronize()
    ref = F.layer_norm(xd, (Cc,), gamma.double().cpu(), beta.double().cpu(), 1e-5)
    rstd = 1.0 / (xd.var(-1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    dmean = (2 * ni + 6) * U32 * xd.abs().mean(-1, keepdim=True)
    bound = dmean * rstd * gamma.double().abs().cpu() + 2.0 ** -16 * ref.abs() \
        + 2.0 ** -18 * (beta.double().abs().cpu() + 1)
    assert excess(y.value(), ref, bound) <= 1.0
    assert y.sentinel_intact()
    # RMSNorm: relative error of mean(x^2) <= (4 NI + 6) 2^-24 (4 NI sequential terms per lane, 5 butterfly steps),
    # halved by the square root, + rsqrtf (2 ulp) and two products; the lo half adds 2^-17
    yr = Out(rows, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 4, ld=2 * Cc + 12)
    yf = Out(rows, Cc, dtype=torch.float32, device=cuda, ld=Cc, row_pad=4)
    L.rmsnorm(x, gamma, 1e-6, yr.view, split_off=yr.split_off, y_f32=yf.buf[:rows])
    torch.cuda.synchronize()
    refr = gamma.double().cpu() * xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6)
    rel = (2 * ni + 10) * U32
    assert excess(yr.value(), refr, (rel + 2.0 ** -16) * refr.abs() + 1e-30) <= 1.0
    assert excess(yf.hi, refr, rel * refr.abs() + 1e-30) <= 1.0
    assert yr.sentinel_intact() and yf.sentinel_intact()


# ---------------------------------------------------------------------------------------------------- T5 front end
def test_gather_rows_ids_edges(cuda):
    """tng_gather_rows bit for bit: ids 0, n - 1 and repeats, 21 rows (not a multiple of the 8 rows per CTA), the table
    between NaN rows (a wrong row index reads NaN) and the rows past the output's end kept at the sentinel."""
    g = torch.Generator().manual_seed(21)
    n, C, rows = 50, 36, 21
    tb = torch.full((n + 2, C), NAN)
    tb[1:n + 1] = rand(g, n, C)
    table = tb.to(cuda)[1:n + 1]
    ids = torch.tensor([0, n - 1, 7, 7, 0, n - 1] + torch.randint(0, n, (rows - 6,), generator=g).tolist())
    out = Out(rows, C, dtype=torch.float32, device=cuda, ld=C, row_pad=3)
    L.gather_rows(table, ids.to(cuda), out.buf[:rows])
    torch.cuda.synchronize()
    assert torch.equal(out.hi.cpu(), table.cpu()[ids])
    assert out.sentinel_intact()


FMIN = torch.finfo(torch.float32).min   # the T5 extended attention mask value


def rel_attn_ref(q, k, v, relbias, kbias, *, batch, heads, L):
    """fp64 T5 self-attention softmax(q k^T + relbias[h, key - query + L - 1] + kbias[b, key]) v (no scaling) of
    q / k / v [batch * L, heads * 64]. Also returns sum p |v| and the per-query score allowance: max over the live keys
    of 2^-24 (64 sum_d |q_d k_d| + 4 |s|) (the fp32 fma chain over 64 dims, the bias add and s - max)."""
    sh = lambda t: t.double().reshape(batch, L, heads, 64).transpose(1, 2)
    qh, kh, vh = sh(q), sh(k), sh(v)
    pos = torch.arange(L)
    s = qh @ kh.transpose(-1, -2) + relbias.double()[:, pos[None, :] - pos[:, None] + L - 1][None]
    live = torch.ones(batch, 1, 1, L, dtype=torch.bool)
    if kbias is not None:
        s = s + kbias.double().view(batch, 1, 1, L)
        live = kbias.view(batch, 1, 1, L) > FMIN
    p = s.softmax(-1)
    ds = U32 * (64 * (qh.abs() @ kh.abs().transpose(-1, -2)) + 4 * s.abs())
    ds = ds.masked_fill(~live, 0.0).amax(-1, keepdim=True).expand(-1, -1, -1, 64)
    back = lambda t: t.transpose(1, 2).reshape(batch * L, heads * 64)
    return back(p @ vh), back(p @ vh.abs()), back(ds)


def rel_attn_bound(pv, ds, L_):
    """A score error d moves the output by <= 2 d sum p |v|. The softmax arithmetic (u = 2^-24): the PV fma chain runs
    over all L keys (L u), l takes 8 roundings per 64-key tile (pair sum, 5 butterfly steps, rescale, add), o one
    rescale per tile, expf 2 ulp (4 u), 1 / l and the final product 2 u: (L + 9 ceil(L / 64) + 6) u <= 2 (L + 70) u of
    sum p |v| for every L."""
    return (2 * ds + 2 * (L_ + 70) * U32) * pv


def rel_attn_operands(g, B, heads, L_, *, grow=False):
    """q / k / v fp32 [B * L, heads * 64] and a relative bias [heads, 2L - 1] with a large, asymmetric spread (it rises
    from -6 to +3 with key - query, plus N(0, 2^2)): a query - key index instead of key - query changes every row.
    grow: key magnitudes rise 0.2 -> 2.5 along the sequence, so the running maximum moves in later key tiles."""
    inner = heads * 64
    q, k, v = (rand(g, B * L_, inner, scale=0.5) for _ in range(3))
    v += 0.3
    if grow:
        k *= torch.linspace(0.2, 2.5, L_).repeat(B)[:, None]
    relbias = rand(g, heads, 2 * L_ - 1, scale=2.0) + torch.linspace(-6.0, 3.0, 2 * L_ - 1)
    return q, k, v, relbias


def rel_attn_kbias(B, L_, mode):
    """None, or an additive key mask of 0 / finfo.min: 'tail' masks the last b + 1 keys of sequence b, 'all but key 0'
    every key but the first, 'one sequence' every key of sequence 1 (and a tail of sequence 0)."""
    if mode is None:
        return None
    kb = torch.zeros(B, L_)
    if mode == "tail":
        for b in range(B):
            kb[b, L_ - b - 1:] = FMIN
    elif mode == "all but key 0":
        kb[:, 1:] = FMIN
    else:
        kb[0, L_ - 3:] = FMIN
        kb[1, :] = FMIN
    return kb


REL_CASES = [(1, 1, 1, None, True, False), (3, 2, 5, "tail", False, False), (2, 16, 16, None, True, False),
             (3, 1, 17, "all but key 0", True, False), (2, 2, 64, "tail", True, False),
             (3, 16, 65, "one sequence", False, False), (2, 2, 129, None, True, True),
             (3, 1, 129, "one sequence", True, True)]


@pytest.mark.parametrize("B,heads,L_,mask,split,grow", REL_CASES)
def test_rel_attention_sequence_edges(cuda, B, heads, L_, mask, split, grow):
    """tng_rel_attention at L = 1, 5, 16, 17, 64, 65, 129 (the 16-query CTA, 4 queries per warp, 64-key tiles) with
    heads 1 / 2 / 16: q / k / v at non-zero, out-of-order columns (v, k, q) of one NaN-padded fp32 buffer with
    ld > 3 * inner, relbias and kbias inside NaN padding, an output at a column offset (bf16, or hi/lo with a gap).
    Against fp64 on the fp32 operands, per element. A fully masked sequence: every score absorbs into finfo.min alike
    (in fp32 and in fp64), so its rows are the uniform mean of V."""
    g = torch.Generator().manual_seed(B * 1000 + heads * 10 + L_)
    inner = heads * 64
    q, k, v, relbias = rel_attn_operands(g, B, heads, L_, grow=grow)
    kb = rel_attn_kbias(B, L_, mask)
    cols = {"v": 8, "k": 8 + inner + 4, "q": 8 + 2 * inner + 12}
    buf = torch.full((B * L_ + 3, 3 * inner + 32), NAN)
    for name, t in (("q", q), ("k", k), ("v", v)):
        buf[:B * L_, cols[name]:cols[name] + inner] = t
    qkv = buf.to(cuda)[:B * L_]
    out = Out(B * L_, inner, dtype=torch.bfloat16, device=cuda, col0=4, split_off=inner + 8 if split else 0,
              ld=2 * inner + 24)
    L.rel_attention(qkv, poisoned_flat(relbias.reshape(-1).to(cuda), lead=3),
                    None if kb is None else poisoned_flat(kb.reshape(-1).to(cuda), lead=1), out.view, batch=B,
                    heads=heads, L=L_, q_col0=cols["q"], k_col0=cols["k"], v_col0=cols["v"], split_off=out.split_off)
    torch.cuda.synchronize()
    ref, pv, ds = rel_attn_ref(q, k, v, relbias, kb, batch=B, heads=heads, L=L_)
    bound = rel_attn_bound(pv, ds, L_)
    e = excess(out.hi, ref, bound + 2.0 ** -8 * ref.abs())
    if split:
        e = max(e, excess(out.value(), ref, bound + 2.0 ** -16 * ref.abs()))
    print(f"rel_attention B={B} heads={heads} L={L_} mask={mask} {'hi/lo' if split else 'bf16'}: worst excess {e:.3f}")
    assert e <= 1.0
    assert out.sentinel_intact()
    if mask == "one sequence":
        mean_v = v.double().view(B, L_, inner)[1].mean(0)
        assert el_err(ref.view(B, L_, inner)[1], mean_v.expand(L_, -1)) < 1e-12
    if mask == "all but key 0":          # p = (1, 0, ...) exactly: the rows are key 0's value row
        want = bf(v.view(B, L_, inner)[:, :1].expand(B, L_, inner).reshape(B * L_, inner))
        assert torch.equal(out.hi.cpu(), want)


# ---------------------------------------------------------------------------------------------------- small kernels
def test_cast_act_upsample_hi_lo_ld(cuda):
    """tng_cast_act with ld_x > C, nearest x2 upsample, leaky-ReLU and a hi/lo output with a gap: bit for bit."""
    g = torch.Generator().manual_seed(3)
    NB, H, W, Cc = 2, 5, 3, 36
    x = poisoned(rand(g, NB * H * W, Cc, scale=3.0).to(cuda), col_pad=8, align=4)
    y = Out(NB * 4 * H * W, Cc, dtype=torch.bfloat16, device=cuda, split_off=Cc + 8, ld=2 * Cc + 16)
    yc = y.cpu_clone()
    S.spec_cast_act(x.cpu(), NB, H, W, yc.view, upsample2x=True, act=L.ACT_LRELU, act_param=0.1, split_off=y.split_off)
    L.cast_act(x, NB, H, W, y.view, upsample2x=True, act=L.ACT_LRELU, act_param=0.1, split_off=y.split_off)
    torch.cuda.synchronize()
    assert torch.equal(y.buf.cpu(), yc.buf)


@pytest.mark.parametrize("Lr", [1, 255, 257, 1000])
def test_softmax_rows_lengths(cuda, Lr):
    """tng_softmax_rows at L = 1, 255, 257 (one past the block), 1000, with ld_x > L and a hi/lo output: against fp64
    (hi + lo: 2^-17 relative; expf and an fp32 sum over <= 1000 terms in a few levels: ~2^-20)."""
    g = torch.Generator().manual_seed(Lr)
    rows = 19
    x = poisoned(rand(g, rows, Lr, scale=4.0).to(cuda), col_pad=5, align=1)
    y = Out(rows, Lr, dtype=torch.bfloat16, device=cuda, split_off=Lr + 3, ld=2 * Lr + 9)
    L.softmax_rows(x, 0.7, y.view, L=Lr, split_off=y.split_off)
    torch.cuda.synchronize()
    ref = (x.double().cpu() * 0.7).softmax(-1)
    assert excess(y.value(), ref, 2.0 ** -16 * ref + 1e-30) <= 1.0
    assert y.sentinel_intact()


@pytest.mark.parametrize("B,R,Cc", [(3, 70, 45), (2, 33, 100), (1, 1, 31)])
def test_transpose_ragged(cuda, B, R, Cc):
    """tng_transpose_bf16 with R, C not multiples of the 32 x 32 tile, ld_x > C and ld_y > R: bit for bit."""
    g = torch.Generator().manual_seed(R * Cc)
    x = poisoned(bf(rand(g, B * R, Cc)).to(cuda), col_pad=3, align=1)
    y = Out(B * Cc, R, dtype=torch.bfloat16, device=cuda, ld=R + 5)
    yc = y.cpu_clone()
    S.spec_transpose_bf16(x.cpu(), B, R, Cc, yc.view)
    L.transpose_bf16(x, B, R, Cc, y.view)
    torch.cuda.synchronize()
    assert torch.equal(y.buf.cpu(), yc.buf)


@pytest.mark.parametrize("rate,ktaps", [(5, 16), (4, 16), (2, 8), (2, 4)])
def test_convt_gather_hifigan_rates(cuda, rate, ktaps):
    """tng_convt_gather at the HiFi-GAN (rate, kernel) pairs, every output position including the first and the last,
    against spec_convt_gather (fp64) and F.conv_transpose1d; at most ceil(k / rate) + 1 fp32 adds per element."""
    g = torch.Generator().manual_seed(rate * 100 + ktaps)
    B, Lin, Cout = 2, 23, 32
    pad = (ktaps - rate) // 2
    Lout = (Lin - 1) * rate - 2 * pad + ktaps
    Y = rand(g, B * Lin, ktaps * Cout).to(cuda)
    bias = rand(g, Cout).to(cuda)
    y = Out(B * Lout, Cout, dtype=torch.float32, device=cuda, ld=Cout, row_pad=3)
    L.convt_gather(Y, B, Lin, ktaps, Cout, rate, pad, Lout, bias, y.buf[:B * Lout])
    torch.cuda.synchronize()
    ref = torch.empty(B * Lout, Cout)
    S.spec_convt_gather(Y.cpu(), B, Lin, ktaps, Cout, rate, pad, Lout, bias.cpu(), ref)
    absref = torch.empty(B * Lout, Cout)
    S.spec_convt_gather(Y.cpu().abs(), B, Lin, ktaps, Cout, rate, pad, Lout, bias.cpu().abs(), absref)
    nadd = -(-ktaps // rate) + 1
    assert excess(y.hi, ref, (nadd + 1) * U32 * absref.double() + 1e-30) <= 1.0
    # the spec itself against torch's transposed convolution (weights = identity taps)
    Yv = Y.cpu().double().view(B, Lin, ktaps, Cout)
    xin = Yv.permute(0, 3, 2, 1).reshape(B, Cout * ktaps, Lin)
    wt = torch.zeros(Cout * ktaps, Cout, ktaps, dtype=torch.float64)
    for co in range(Cout):
        for t in range(ktaps):
            wt[co * ktaps + t, co, t] = 1.0
    tref = F.conv_transpose1d(xin, wt, bias.cpu().double(), stride=rate, padding=pad).permute(0, 2, 1).reshape(-1, Cout)
    assert el_err(ref, tref) < 1e-6
    assert y.sentinel_intact()


def test_tanh_to_i16_edges(cuda):
    """tng_tanh_to_i16: +-inf, +-20 (tanh = +-1.0: +1.0 * 32768 wraps to -32768, as numpy's astype does), small values,
    read with ld_x = 3 from a NaN-padded buffer: bit for bit against spec_tanh_to_i16."""
    vals = torch.tensor([math.inf, -math.inf, 20.0, -20.0, 0.0, 0.5, -0.5, 1e-3, -1e-3, 2.0, -3.7, 0.25])
    n, ld = vals.numel(), 3
    xb = torch.full((n * ld + 2,), NAN)
    xb[:n * ld:ld] = vals
    x = xb.to(cuda)
    wf = Out(1, n, dtype=torch.float32, device=cuda, row_pad=1)
    wi = torch.full((n + 5,), 12345, dtype=torch.int16, device=cuda)
    L.tanh_to_i16(x, n, ld, wf.buf[0, :n], wi[:n])
    torch.cuda.synchronize()
    ef, ei = torch.empty(n), torch.empty(n, dtype=torch.int16)
    S.spec_tanh_to_i16(xb, n, ld, ef, ei)
    assert torch.equal(wi[:n].cpu(), ei) and (wi[n:] == 12345).all()
    assert ei[0].item() == -32768 and ei[2].item() == -32768 and ei[3].item() == -32768   # +1.0 wraps
    assert excess(wf.hi[0], ef, 4 * U32 * ef.abs() + 1e-45) <= 1.0    # tanhf: within 2 ulp
    assert wf.sentinel_intact()


@pytest.mark.parametrize("dim,flip", [(321, True), (65, False), (320, True)])
def test_timestep_embedding_odd_dim_freq_shift(cuda, dim, flip):
    """tng_timestep_embedding with odd dim (the last column is zero) and freq_shift = 1, against an fp64 evaluation of
    the fp32 exponent table (|t| <= 999: the fp32 argument t * exp(.) is off by up to ~2 ulp(999) ~ 1.2e-4)."""
    t = torch.tensor([0.0, 1.0, 37.0, 500.0, 999.0])
    n, half = t.numel(), dim // 2
    out = Out(n, dim, dtype=torch.float32, device=cuda, ld=dim, row_pad=2)
    L.timestep_embedding(t.to(cuda), dim, flip, 1.0, out.buf[:n])
    torch.cuda.synchronize()
    e = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / (half - 1.0)).double()
    a = t.double()[:, None] * e[None, :]
    parts = [torch.cos(a), torch.sin(a)] if flip else [torch.sin(a), torch.cos(a)]
    ref = torch.cat(parts + ([torch.zeros(n, 1, dtype=torch.float64)] if dim % 2 else []), dim=-1)
    assert excess(out.hi, ref, 2.5e-4) <= 1.0
    if dim % 2:
        assert (out.hi[:, -1] == 0).all()
    assert out.sentinel_intact()


# ---------------------------------------------------------------------------------------------------- tng_linear_f32
def silu64(x):
    return x * torch.sigmoid(x)


def linear_f32_reference(x, w, b, pre, post):
    """fp64 post(pre(x) w^T + b) and its per-element allowance (u = 2^-24): each lane sums ceil(K/32) products in one fma
    chain, then 5 butterfly steps and the bias add: (ceil(K/32) + 6) u sum |a w| (+ |b|). The sm_90 SiLU (ex2 2 ulp, rcp
    1 ulp, two roundings, and the rounding of its exponent argument: |x| u) is within (8 + |x|) u relative; |silu'| <= 1.1."""
    x, w = x.double(), w.double()
    bd = 0.0 if b is None else b.double()
    a = silu64(x) if pre == L.ACT_SILU else x
    y = a @ w.t() + bd
    err = (math.ceil(x.shape[1] / 32) + 6) * U32 * (a.abs() @ w.abs().t() + abs(bd))
    if pre == L.ACT_SILU:
        err = err + U32 * (((8 + x.abs()) * a.abs()) @ w.abs().t())
    if post == L.ACT_SILU:
        z = silu64(y)
        return z, 1.1 * err + U32 * (8 + y.abs()) * z.abs()
    return y, err


def linear_f32_operands(g, device, M, K, N, has_b):
    """x [M, K], w [N, K] (dense, followed by NaN) and b [N] (inside NaN padding) or None."""
    x = poisoned_flat(rand(g, M * K, scale=2.0).to(device)).view(M, K)
    w = poisoned_flat(rand(g, N * K, scale=K ** -0.5).to(device)).view(N, K)
    return x, w, poisoned_flat(rand(g, N).to(device), lead=2) if has_b else None


@pytest.mark.parametrize("pre,post", [(L.ACT_NONE, L.ACT_NONE), (L.ACT_NONE, L.ACT_SILU), (L.ACT_SILU, L.ACT_NONE),
                                      (L.ACT_SILU, L.ACT_SILU)])
def test_linear_f32_shapes_and_activations(cuda, pre, post):
    """tng_linear_f32 over M in {1, 5}, K in {31, 32, 320} (a partial lane stride, one stride, ten), N in {1, 7, 1280},
    with and without a bias: per element against fp64, the rows past M kept at the sentinel."""
    g = torch.Generator().manual_seed(pre * 2 + post)
    worst = 0.0
    for M in (1, 5):
        for K in (31, 32, 320):
            for N in (1, 7, 1280):
                for has_b in (False, True):
                    x, w, b = linear_f32_operands(g, cuda, M, K, N, has_b)
                    y = Out(M, N, dtype=torch.float32, device=cuda, ld=N, row_pad=2)
                    L.linear_f32(x, w, b, y.buf[:M], pre_act=pre, post_act=post)
                    torch.cuda.synchronize()
                    ref, bound = linear_f32_reference(x.cpu(), w.cpu(), None if b is None else b.cpu(), pre, post)
                    e = excess(y.hi, ref, bound)
                    worst = max(worst, e)
                    assert e <= 1.0 and y.sentinel_intact(), (M, K, N, has_b, e)
    print(f"linear_f32 pre={pre} post={post}: worst excess {worst:.3f}")


# ---------------------------------------------------------------------------------------------------- mel front end
FLOOR = 1e-5


def ulp32(r):
    """The fp32 ulp at each value of r (as fp64)."""
    a = r.float().abs()
    return (torch.nextafter(a, torch.tensor(math.inf)) - a).double()


@pytest.mark.parametrize("pad,T", [(64, 65), (64, 131), (512, 513), (512, 1027)])
def test_stft_frames_reflect_edges(cuda, pad, T):
    """tng_stft_frames bit for bit against spec_stft_frames at T = pad + 1 (the shortest legal reflect) and T = 2 pad + 3,
    B = 3, ld = T + 2 pad + 13: both planes entirely (the zero tail past T + 2 pad is written), rows past B untouched;
    the waveform is followed by NaN."""
    g = torch.Generator().manual_seed(pad + T)
    B, ld = 3, T + 2 * pad + 13
    y = poisoned_flat(rand(g, B * T, scale=0.5).to(cuda)).view(B, T)
    hi, lo = (Out(B, ld, dtype=torch.bfloat16, device=cuda, ld=ld, row_pad=2) for _ in range(2))
    hc, lc = hi.cpu_clone(), lo.cpu_clone()
    S.spec_stft_frames(y.cpu(), pad, hc.buf[:B], lc.buf[:B])
    L.stft_frames(y, pad, hi.buf[:B], lo.buf[:B])
    torch.cuda.synchronize()
    assert torch.equal(hi.buf.cpu(), hc.buf) and torch.equal(lo.buf.cpu(), lc.buf)
    assert (hc.buf[:B, T + 2 * pad:] == 0).all() and (lc.buf[:B, T + 2 * pad:] == 0).all()


@pytest.mark.parametrize("null_out", ["mag", "log_mag", "energy"])
@pytest.mark.parametrize("bins", [17, 32, 33, 513])
def test_stft_magnitude_layout_and_bounds(cuda, bins, null_out):
    """tng_stft_magnitude with ldF > 2 bins (NaN past column 2 bins), 13 rows (not a multiple of the 8 warps), all-zero
    frames and frames below the floor, each output NULL in turn. The magnitude is sqrt(rn(rn(re^2) + rn(im^2))), one IEEE
    op per step on both sides: the operand is bit-exact against spec_stft_magnitude in the model's layout (hi at column 0,
    lo at c_pad > bins; the pad columns [bins, c_pad) keep their sentinel: the mel GEMM reads them against zero weights).
    log_mag within 1 ulp of the fp64 log (CUDA's documented logf bound); energy: an fma chain of ceil(bins / 32) per lane
    and 5 butterfly steps, halved by the square root, + its rounding: ((ceil(bins/32) + 6) / 2 + 1) 2^-24 relative."""
    g = torch.Generator().manual_seed(bins * 3 + len(null_out))
    rows = 13
    c_pad = (bins + 1 + 7) // 8 * 8
    Fq = rand(g, rows, 2 * bins, scale=3.0)
    Fq[[2, 9]] = 0.0                   # silent frames: log(floor)
    Fq[5] *= 1e-7                      # below the floor
    Fd = poisoned(Fq.to(cuda), col_pad=5, align=1)
    mag = None if null_out == "mag" else Out(rows, bins, dtype=torch.bfloat16, device=cuda, split_off=c_pad,
                                             ld=2 * c_pad + 8)
    logm = None if null_out == "log_mag" else Out(rows, bins, dtype=torch.float32, device=cuda, ld=bins, row_pad=2)
    en = None if null_out == "energy" else Out(rows, 1, dtype=torch.float32, device=cuda, ld=1, row_pad=3)
    L.stft_magnitude(Fd, bins, None if mag is None else mag.view, c_pad, None if logm is None else logm.buf[:rows],
                     None if en is None else en.buf[:rows, 0], FLOOR)
    torch.cuda.synchronize()
    m = torch.sqrt((Fq[:, :bins] * Fq[:, :bins] + Fq[:, bins:] * Fq[:, bins:]).double()).float()   # as the spec
    if mag is not None:
        mc = mag.cpu_clone()
        S.spec_stft_magnitude(Fd.cpu(), bins, mc.view, c_pad, None, None, FLOOR)
        assert torch.equal(mag.buf.cpu(), mc.buf)
    msg = [f"stft_magnitude bins={bins} ({null_out} NULL):"]
    if logm is not None:
        ref = torch.log(torch.clamp(m.double(), min=torch.tensor(FLOOR, dtype=torch.float32).item()))
        e = excess(logm.hi, ref, ulp32(ref))
        msg.append(f"log_mag worst excess {e:.3f}")
        assert e <= 1.0 and logm.sentinel_intact()
        silent = logm.hi[[2, 9]].cpu()
        assert (silent == silent[0, 0]).all()       # the same log(floor) everywhere
    if en is not None:
        ref = m.double().pow(2).sum(1).sqrt()
        e = excess(en.hi[:, 0], ref, ((math.ceil(bins / 32) + 6) / 2 + 1) * U32 * ref + 1e-45)
        msg.append(f"energy worst excess {e:.3f}")
        assert e <= 1.0 and en.sentinel_intact()
    print(" ".join(msg))


def test_log_clamp_edges(cuda):
    """tng_log_clamp on values below, at and just above the floor, 0, -0, negatives, denormals, +inf and a spread of
    magnitudes; n = 1037 (not a multiple of 256) with a sentinel tail: every result within 1 ulp of the fp64
    log(max(x, floor)), +inf to +inf."""
    fl = torch.tensor(FLOOR, dtype=torch.float32)
    special = torch.cat([torch.tensor([0.0, -0.0, -1.0, -1e30, 1e-45, 1e-40, 1.2e-38, 1.0, 2.5, 1e30, math.inf]),
                         (fl * 0.999).view(1), fl.view(1), torch.nextafter(fl, torch.tensor(1.0)).view(1)])
    g = torch.Generator().manual_seed(5)
    x = torch.cat([special, torch.exp(rand(g, 1037 - special.numel(), scale=8.0))]).float()
    n = x.numel()
    y = Out(1, n, dtype=torch.float32, device=cuda, ld=n, row_pad=1)
    L.log_clamp(poisoned_flat(x.to(cuda)), y.buf[0], FLOOR)
    torch.cuda.synchronize()
    ref = torch.log(torch.clamp(x.double(), min=fl.item()))
    got = y.hi[0].cpu()
    fin = torch.isfinite(ref)
    e = excess(got[fin], ref[fin], ulp32(ref[fin]))
    print(f"log_clamp: worst excess {e:.3f}")
    assert e <= 1.0 and (got[~fin] == math.inf).all() and int((~fin).sum()) == 1
    assert y.sentinel_intact()
