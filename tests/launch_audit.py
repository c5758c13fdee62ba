"""Per-launch audit of the kernels the product itself issues (TEST INFRASTRUCTURE ONLY).

`install_audit(monkeypatch)` wraps every kernel wrapper of tango_b200.lib, so that a real generation (or, with the spec
backend of cabi_spec.py installed first, its CPU statement) checks each launch against its C-ABI contract with the
launch's own descriptor, buffers and inputs:

  1. snapshot: every storage the call may write is copied (outputs, read-modify-write accumulators, inputs aliased to an
     output: `res` = `out_f32`, `accumulate`, the GroupNorm statistics, `last`, a masked blend's `sample`);
  2. poison: the contract's output region is filled with NaN (int16: a sentinel) wherever the call does not read it, so
     an element the kernel never writes fails;
  3. run the wrapper, synchronise, evaluate the reference on the snapshot (on the tensors' device, in fp64 where the
     contract is approximate, with the per-element bounds of test_kernel_contract_gpu.py);
  4. every byte of the written storages outside the contract region (hi/lo gaps, ld padding, neighbouring buffers
     carved from the same storage) must equal the snapshot bit for bit;
  5. record (entry point, plan family, shape, worst excess); a launch over its bound raises at once, naming itself.

It checks kernels against their descriptors; whether the host builds the right descriptors is the business of
test_orchestration_spec.py and the parity tests.
"""
from __future__ import annotations

import inspect
import math
from collections import defaultdict
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

import cabi_spec as S
from tango_b200 import lib as L
from test_kernel_contract_gpu import (U32, act_ref, attn_ref, flat_base, geglu_reference, gemm_gamma,
                                      linear_f32_reference, rel_attn_bound, rel_attn_ref, ulp32)
from unipc_spec import spec_unipc_step

SPECS = dict(S.SPEC, unipc_step=spec_unipc_step)
ENTRY_POINTS = tuple(sorted(SPECS))
LATENT_STEPS = ("sched_step", "dpm_step", "unipc_step", "latent_blend")
I16_POISON = -12345
SCORE_BUDGET = 2 ** 28      # fp64 score elements per attention reference chunk (2 GB)


class AuditFailure(AssertionError):
    pass


@dataclass
class Record:
    index: int
    entry: str
    family: str
    shape: str
    excess: float
    launches: int
    tags: frozenset = field(default_factory=frozenset)
    work: int = 0           # grid-stride walk length of the elementwise kernels (latent steps: elements, cast_act: quads)


# ---------------------------------------------------------------------------------------------------- contract regions
def _hilo(t, rows, cols, split_off):
    if t is None:
        return []
    return [t[:rows, :cols]] + ([t[:rows, split_off:split_off + cols]] if split_off else [])


def _flat_n(t, n):
    return [] if t is None else [t.reshape(-1)[:n]]


def _whole(t):
    return [] if t is None else [t]


def _gemm_width(a):
    N = a["weight"].shape[0]
    return N // 2 if a["act"] in (L.ACT_GEGLU, L.ACT_GEGLU_TANH) else N


def _next_in(a):
    return ("next_in", _hilo(a["next_in"], (2 if a["cfg"] else 1) * a["B"] * a["HW"], a["Cc"], a["split_off"]), False)


# entry -> bound arguments -> [(argument, [region views], read by the call)]
REGIONS = {
    "conv_gemm": lambda a: [
        ("out_f32", _hilo(a["out_f32"], a["NB"] * a["H"] * a["W"], a["weight"].shape[0], 0), a["accumulate"]),
        ("out_bf16", _hilo(a["out_bf16"], a["NB"] * a["H"] * a["W"], _gemm_width(a), a["split_off"]), False),
        ("gn_stats", _whole(a["gn_stats"]), True)],
    "attention": lambda a: [("out", _hilo(a["out"], a["batch"] * a["Lq"], a["heads"] * 64, a["split_off"]), False)],
    "attention_wide": lambda a: [("out", _hilo(a["out"], a["batch"] * a["L"], a["dim"], 0), False)],
    "rel_attention": lambda a: [("out", _hilo(a["out"], a["batch"] * a["L"], a["heads"] * 64, a["split_off"]), False)],
    "groupnorm_stats": lambda a: [("stats", _whole(a["stats"]), True)],
    "groupnorm": lambda a: [
        ("y", _hilo(a["y"], a["NB"] * a["HW"], _gn_channels(a), a["split_off"]), False),
        ("raw", _hilo(a["raw"], a["NB"] * a["HW"], _gn_channels(a), a["raw_split_off"]), False)],
    "layernorm": lambda a: [("y", _hilo(a["y"], *a["x"].shape, a["split_off"]), False)],
    "rmsnorm": lambda a: [("y", _hilo(a["y"], *a["x"].shape, a["split_off"]), False), ("y_f32", _whole(a["y_f32"]), False)],
    "gather_rows": lambda a: [("out", _whole(a["out"]), False)],
    "cast_act": lambda a: [("y", _hilo(a["y"], a["NB"] * a["H"] * a["W"] * (4 if a["upsample2x"] else 1),
                                       a["x"].shape[-1] if a["Cc"] is None else a["Cc"], a["split_off"]), False)],
    "softmax_rows": lambda a: [("y", _hilo(a["y"], a["x"].shape[0], a["x"].shape[1] if a["L"] is None else a["L"],
                                           a["split_off"]), False)],
    "transpose_bf16": lambda a: [("y", _hilo(a["y"], a["B"] * a["Cc"], a["R"], 0), False)],
    "sched_step": lambda a: [("prev", _flat_n(a["prev"], a["B"] * a["Cc"] * a["HW"]), False), _next_in(a)],
    "dpm_step": lambda a: [("m0", _flat_n(a["m0"], a["B"] * a["Cc"] * a["HW"]), False),
                           ("prev", _flat_n(a["prev"], a["B"] * a["Cc"] * a["HW"]), False), _next_in(a)],
    "unipc_step": lambda a: [("m_cur", _flat_n(a["m_cur"], a["B"] * a["Cc"] * a["HW"]), False),
                             ("last", _flat_n(a["last"], a["B"] * a["Cc"] * a["HW"]), a["corrector_order"] > 0),
                             ("prev", _flat_n(a["prev"], a["B"] * a["Cc"] * a["HW"]), False), _next_in(a)],
    "latent_blend": lambda a: [("sample", _flat_n(a["sample"], a["B"] * a["Cc"] * a["HW"]), a["mask"] is not None),
                               _next_in(a)],
    "timestep_embedding": lambda a: [("out", _whole(a["out"]), False)],
    "linear_f32": lambda a: [("y", _whole(a["y"]), False)],
    "convt_gather": lambda a: [("y", _whole(a["y"]), False)],
    "tanh_to_i16": lambda a: [("wave_f32", _flat_n(a["wave_f32"], a["n"]), False),
                              ("wave_i16", _flat_n(a["wave_i16"], a["n"]), False)],
    "stft_frames": lambda a: [("hi", _whole(a["hi"]), False), ("lo", _whole(a["lo"]), False)],
    "stft_magnitude": lambda a: [("mag_op", _hilo(a["mag_op"], a["Fq"].shape[0], a["bins"], a["split_off"]), False),
                                 ("log_mag", _whole(a["log_mag"]), False), ("energy", _whole(a["energy"]), False)],
    "log_clamp": lambda a: [("y", _whole(a["y"]), False)],
}


def _gn_channels(a):
    return a["x0"].shape[-1] + (0 if a["x1"] is None else a["x1"].shape[-1])


# ---------------------------------------------------------------------------------------------------- storages
def _skey(t):
    return (t.device, t.untyped_storage().data_ptr())


def _storage_1d(t):
    """The whole storage of t as a 1-D tensor of t's dtype."""
    st = t.untyped_storage()
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(st, 0, (st.nbytes() // t.element_size(),), (1,))


def _mark(mask, t):
    mask.as_strided(t.shape, t.stride(), t.storage_offset()).fill_(True)


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


class _Storage:
    """One storage the call writes: its snapshot and the element masks of the contract region and of what is read."""

    def __init__(self, t):
        self.live = _storage_1d(t)
        self.snap = self.live.clone()
        self.region = torch.zeros(self.live.numel(), dtype=torch.bool, device=t.device)
        self.read = torch.zeros_like(self.region)

    def remap(self, t):
        """t (a view of this storage) as the same view of the snapshot."""
        assert t.dtype == self.live.dtype, "a storage written under two dtypes"
        return self.snap.as_strided(t.shape, t.stride(), t.storage_offset())


def _tensors(v):
    if isinstance(v, torch.Tensor):
        yield v
    elif isinstance(v, L.View):
        yield v.t
    elif isinstance(v, (list, tuple)):
        for x in v:
            yield from _tensors(x)


def _read_extents(v):
    """The tensors an argument reads; an activation view: only its (NB, H, W, C) extent, not its whole buffer."""
    if isinstance(v, L.View):
        yield v.t.as_strided((v.NB, v.H, v.W, v.C), (v.s_n, v.s_h, v.s_w, 1), v.t.storage_offset() + v.off)
    elif isinstance(v, (list, tuple)):
        for x in v:
            yield from _read_extents(x)
    elif isinstance(v, torch.Tensor):
        yield v


def _remap_arg(v, stores):
    if isinstance(v, torch.Tensor):
        s = stores.get(_skey(v))
        return v if s is None else s.remap(v)
    if isinstance(v, L.View):
        return L.View(_remap_arg(v.t, stores), v.C, v.W, v.H, v.NB, v.s_w, v.s_h, v.s_n, v.off)
    if isinstance(v, list):
        return [_remap_arg(x, stores) for x in v]
    if isinstance(v, tuple):
        return tuple(_remap_arg(x, stores) for x in v)
    return v


# ---------------------------------------------------------------------------------------------------- checks
def _excess(got, ref, bound) -> float:
    """max |got - ref| / bound (inf on a non-finite value where the reference is finite)."""
    got, ref = got.double(), ref.double()
    if got.numel() == 0:
        return 0.0
    if not torch.isfinite(got).all():
        return math.inf
    return ((got - ref).abs() / bound.double().clamp_min(1e-300)).max().item()


def _val(t, rows, cols, split_off):
    """(hi, hi + lo or None) of a bf16 output region."""
    hi = t[:rows, :cols]
    return hi, (hi.double() + t[:rows, split_off:split_off + cols].double()) if split_off else None


def _rounded(out, ref, bound, split_off, rows, cols):
    """A bf16 output (hi, or hi/lo at split_off) of the value ref within bound + its rounding."""
    hi, val = _val(out, rows, cols, split_off)
    e = _excess(hi, ref, bound + 2.0 ** -8 * ref.abs())
    if val is not None:
        e = max(e, _excess(val, ref, bound + 2.0 ** -16 * ref.abs()))
    return e


def gemm_reference_dev(a, absval=False):
    """spec_conv_gemm of the launch's descriptor on its own device -> fp32-rounded y [rows, Ncols] in fp64; absval: the
    same contraction and epilogue on |operands| (the per-element scale of the fp32 summation error)."""
    f = torch.abs if absval else (lambda t: t)
    views = [L.View(f(flat_base(v.t)), v.C, v.W, v.H, v.NB, v.s_w, v.s_h, v.s_n, v.off) for v in a["views"]]
    rows, N = a["NB"] * a["H"] * a["W"], a["weight"].shape[0]
    acc = bool(a["accumulate"])
    out = f(a["out_f32"][:rows, :N].double()).clone() if acc else \
        torch.zeros(rows, N, dtype=torch.float64, device=a["weight"].device)
    ek = {k: f(a[k]) for k in ("bias", "res") if a[k] is not None}
    if a["rowvec"] is not None:          # pointer + leading dimension: the storage from the first element on
        ek["rowvec"] = f(flat_base(a["rowvec"]))
    alpha = abs(a["alpha"]) if absval else a["alpha"]
    S.spec_conv_gemm(views, a["groups"], f(a["weight"]), a["W"], a["H"], a["NB"], alpha=alpha, accumulate=acc,
                     rowvec_ld=a["rowvec_ld"] or N, out_f32=out, **ek)
    return out


def gemm_stats_bound(o):
    """GroupNorm statistics of the stored output o [images, HW, Ncols] (fp64): fp32 partials over <= 128 rows, fp64
    across partials -> |error| <= 128 * 2^-24 * sum |x| (and sum x^2); as test_gemm_tall_tiles_gpu.run_conv."""
    return 128 * U32 * o.abs().sum(1), 128 * U32 * (o * o).sum(1)


def check_conv_gemm(a, k):
    for name in ("ld_f32", "ld_bf16", "ldr"):
        assert a["_"].get(name) is None, f"conv_gemm: explicit {name} is not audited"
    rows, N = a["NB"] * a["H"] * a["W"], a["weight"].shape[0]
    y = gemm_reference_dev(a)
    ab = gemm_reference_dev(a, absval=True)
    gamma = gemm_gamma(64 * sum(g[5] for g in a["groups"]))
    sb = gamma * ab
    e = 0.0
    if k["out_f32"] is not None:
        e = _excess(k["out_f32"][:rows, :N], y, sb + U32 * y.abs())
    if k["out_bf16"] is not None:
        act = a["act"]
        if act in (L.ACT_GEGLU, L.ACT_GEGLU_TANH):
            z, bound = geglu_reference(y, ab, a["block_n"], act == L.ACT_GEGLU_TANH, gamma=gamma)
        else:
            z, bound = act_ref(y, act, a["act_param"]), (1.1 if act == L.ACT_SILU else 1.0) * sb
        e = max(e, _rounded(k["out_bf16"], z, bound, a["split_off"], rows, z.shape[1]))
    if a["gn_stats"] is not None:
        stored = k["out_f32"][:rows, :N] if k["out_f32"] is not None else k["out_bf16"][:rows, :N]
        o = stored.double().reshape(rows // a["stats_hw"], a["stats_hw"], N)
        d = k["gn_stats"].double() - a["gn_stats"].double()
        b0, b1 = gemm_stats_bound(o)
        e = max(e, _excess(d[..., 0], o.sum(1), b0), _excess(d[..., 1], (o * o).sum(1), b1))
    return e


def _cols(t, col0, lo_off, nsplit, rows, C):
    v = t[:rows, col0:col0 + C].double()
    return v + t[:rows, col0 + lo_off:col0 + lo_off + C].double() if nsplit == 2 else v


def attention_excess(out, split_off, q, k, v, kbias, *, batch, heads, Lq, Lk, scale, nsplit, width=64):
    """Every output element against fp64 attention, one batch entry (and as many heads as fit SCORE_BUDGET) at a time,
    with the bounds of test_kernels_at_scale_gpu.attn_excess: a P rounding error of 2^-7 (bf16 P) or 2^-11 (hi/lo P)
    of sum p |v|, and the output rounding."""
    e = 0.0
    hc = max(1, min(heads, SCORE_BUDGET // (Lq * Lk)))
    pb = 2.0 ** -7 if nsplit == 1 else 2.0 ** -11
    for b in range(batch):
        rq, rk = slice(b * Lq, (b + 1) * Lq), slice(b * Lk, (b + 1) * Lk)
        for h0 in range(0, heads, hc):
            nh = min(hc, heads - h0)
            cs = slice(h0 * width, (h0 + nh) * width)
            ref, pv = attn_ref(q[rq, cs].contiguous(), k[rk, cs].contiguous(), v[rk, cs].contiguous(), batch=1,
                               heads=nh, Lq=Lq, Lk=Lk, scale=scale, width=width,
                               kbias=None if kbias is None else kbias[rk].reshape(1, Lk))
            o = out[rq]
            hi = o[:, cs]
            e = max(e, _excess(hi, ref, pb * pv + 2.0 ** -8 * ref.abs()))
            if split_off:
                val = hi.double() + o[:, split_off + cs.start:split_off + cs.stop].double()
                e = max(e, _excess(val, ref, pb * pv + 2.0 ** -15 * ref.abs()))
    return e


def check_attention(a, k):
    B, H, Lq, Lk, ns = a["batch"], a["heads"], a["Lq"], a["Lk"], a["nsplit"]
    C = H * 64
    q = _cols(a["q"], a["q_col0"], a["q_lo_off"], ns, B * Lq, C)
    kk = _cols(a["k"], a["k_col0"], a["k_lo_off"], ns, B * Lk, C)
    v = _cols(a["v"], a["v_col0"], a["v_lo_off"], ns, B * Lk, C)
    kb = None if a["kbias"] is None else a["kbias"].reshape(-1)[:B * Lk].double()
    return attention_excess(k["out"], a["split_off"], q, kk, v, kb, batch=B, heads=H, Lq=Lq, Lk=Lk,
                            scale=a["scale"], nsplit=ns)


def check_attention_wide(a, k):
    B, L_, D = a["batch"], a["L"], a["dim"]
    q, kk, v = (_cols(a[n], a[n + "_col0"], 0, 1, B * L_, D) for n in ("q", "k", "v"))
    return attention_excess(k["out"], 0, q, kk, v, None, batch=B, heads=1, Lq=L_, Lk=L_, scale=a["scale"], nsplit=1,
                            width=D)


def check_rel_attention(a, k):
    """On the host: T5 sequences are short, and rel_attn_ref builds its position index there."""
    B, H, L_ = a["batch"], a["heads"], a["L"]
    inner = H * 64
    qkv = a["qkv"][:B * L_].cpu()
    q, kk, v = (qkv[:, a[n]:a[n] + inner] for n in ("q_col0", "k_col0", "v_col0"))
    kb = None if a["kbias"] is None else a["kbias"].reshape(-1)[:B * L_].cpu()
    ref, pv, ds = rel_attn_ref(q, kk, v, a["relbias"].cpu(), kb, batch=B, heads=H, L=L_)
    return _rounded(k["out"].cpu(), ref, rel_attn_bound(pv, ds, L_), a["split_off"], B * L_, inner)


def check_groupnorm_stats(a, k):
    NB, HW = a["NB"], a["HW"]
    x = a["x"][:NB * HW].double().view(NB, HW, -1)
    d = k["stats"].double() - a["stats"].double()
    b0, b1 = gemm_stats_bound(x)
    return max(_excess(d[..., 0], x.sum(1), b0), _excess(d[..., 1], (x * x).sum(1), b1))


def check_groupnorm(a, k):
    """The normalisation of the contract with the statistics the launch was given (mean = S / n, var = Q / n - mean^2
    over the group's channels, in fp64 as the kernel takes them). The kernel's fp32 scale / shift (rstd and mean
    rounded to fp32, sc = rstd gamma, sh = beta - mean sc, x sc + sh) is within 4 u (|x| + |mean|) rstd |gamma| + u |beta|
    + 2 u |y|; 2^-20 (16 u) of (|x| + |mean|) rstd |gamma| + |beta| covers it and the SiLU (~2^-21 |y|, |silu'| <= 1.1)."""
    NB, HW, groups = a["NB"], a["HW"], a["groups"]
    rows = NB * HW
    x = a["x0"][:rows].double() if a["x1"] is None else torch.cat([a["x0"][:rows].double(), a["x1"][:rows].double()], 1)
    C_ = x.shape[1]
    st = a["st0"].double() if a["x1"] is None else torch.cat([a["st0"].double(), a["st1"].double()], 1)
    cpg = C_ // groups
    gs = st.view(NB, groups, cpg, 2).sum(2)
    n = float(HW * cpg)
    mean = gs[..., 0] / n
    rstd = 1.0 / torch.sqrt((gs[..., 1] / n - mean * mean).clamp_min(0.0) + a["eps"])
    mc, rc = (t.repeat_interleave(cpg, 1)[:, None, :] for t in (mean, rstd))
    xv = x.view(NB, HW, C_)
    gam, bet = a["gamma"].double(), a["beta"].double()
    y = ((xv - mc) * rc * gam + bet).reshape(rows, C_)
    bound = 2.0 ** -20 * (((xv.abs() + mc.abs()) * rc * gam.abs()).reshape(rows, C_) + bet.abs())
    z = act_ref(y, a["act"])
    e = _rounded(k["y"], z, (1.1 if a["act"] == L.ACT_SILU else 1.0) * bound, a["split_off"], rows, C_)
    if k["raw"] is not None:
        e = max(e, _rounded(k["raw"], x, torch.zeros_like(x), a["raw_split_off"], rows, C_))
    return e


def check_layernorm(a, k):
    """Bounds of test_layernorm_rmsnorm_template_boundaries: the fp32 mean of a lane's 2 NI pairs + 5 butterfly steps
    moves every value by (2 NI + 6) u mean|x| rstd |gamma|; the rest (rstd, the affine, the lo rounding) <= 2^-18."""
    x = a["x"].double()
    rows, Cc = x.shape
    gam, bet = a["gamma"].double(), a["beta"].double()
    ref = F.layer_norm(x, (Cc,), gam, bet, a["eps"])
    rstd = 1.0 / (x.var(-1, unbiased=False, keepdim=True) + a["eps"]).sqrt()
    ni = (Cc // 4 + 31) // 32
    dmean = (2 * ni + 6) * U32 * x.abs().mean(-1, keepdim=True)
    bound = dmean * rstd * gam.abs() + 2.0 ** -18 * (bet.abs() + 1)
    return _rounded(k["y"], ref, bound, a["split_off"], rows, Cc)


def check_rmsnorm(a, k):
    """mean(x^2): (4 NI + 6) u of fp32 sums, halved by the root, + rsqrtf and two products: (2 NI + 10) u relative."""
    x = a["x"].double()
    rows, Cc = x.shape
    ref = a["gamma"].double() * x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + a["eps"])
    rel = (2 * ((Cc // 4 + 31) // 32) + 10) * U32
    e = 0.0
    if k["y"] is not None:
        e = _rounded(k["y"], ref, rel * ref.abs(), a["split_off"], rows, Cc)
    if k["y_f32"] is not None:
        e = max(e, _excess(k["y_f32"], ref, rel * ref.abs() + 1e-30))
    return e


def check_softmax_rows(a, k):
    """hi/lo: 2^-17 of the value + expf and a short fp32 sum (~2^-20); bf16: its rounding on top."""
    L_ = a["x"].shape[1] if a["L"] is None else a["L"]
    ref = (a["x"][:, :L_].double() * a["scale"]).softmax(-1)
    return _rounded(k["y"], ref, 2.0 ** -20 * ref, a["split_off"], ref.shape[0], L_)


def check_timestep_embedding(a, k):
    """fp64 evaluation of the fp32 exponent table; |t| <= 999 puts the fp32 argument within ~2 ulp(999) (2.5e-4)."""
    t = a["t"].double().reshape(-1)
    dim, half = a["dim"], a["dim"] // 2
    ex = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device)
                   / (half - a["freq_shift"])).double()
    ang = t[:, None] * ex[None, :]
    parts = [torch.cos(ang), torch.sin(ang)] if a["flip_sin_to_cos"] else [torch.sin(ang), torch.cos(ang)]
    if dim % 2:
        parts.append(torch.zeros(t.numel(), 1, dtype=torch.float64, device=t.device))
    assert t.abs().max().item() <= 999.0
    ref = torch.cat(parts, -1)
    return _excess(k["out"].reshape(ref.shape), ref, torch.full_like(ref, 2.5e-4))


def check_linear_f32(a, k):
    ref, bound = linear_f32_reference(a["x"], a["w"], a["b"], a["pre_act"], a["post_act"])
    return _excess(k["y"].reshape(ref.shape), ref, bound)


def check_convt_gather(a, k):
    """fp64 overlap-add; at most ceil(k / stride) + 1 fp32 adds per element (the bias included)."""
    B, Lout, Cout = a["B"], a["Lout"], a["Cout"]
    ref, absref = (torch.empty(B * Lout, Cout, dtype=torch.float64, device=a["Y"].device) for _ in range(2))
    args = [a[n] for n in ("B", "Lin", "ktaps", "Cout", "stride", "pad", "Lout")]
    S.spec_convt_gather(a["Y"].double(), *args, None if a["bias"] is None else a["bias"].double(), ref)
    S.spec_convt_gather(a["Y"].double().abs(), *args, None if a["bias"] is None else a["bias"].double().abs(), absref)
    nadd = -(-a["ktaps"] // a["stride"]) + 1
    return _excess(k["y"].reshape(ref.shape), ref, (nadd + 1) * U32 * absref + 1e-30)


def check_tanh_to_i16(a, k):
    """wave_f32 within 2 ulp of tanh (4 u relative); wave_i16 bit for bit the contract's truncation of the fp32 tanh
    the launch produced (of the spec's when it writes no fp32 wave)."""
    n, ld = a["n"], a["ld_x"]
    x = a["x"].reshape(-1)[: n * ld: ld]
    ref = torch.tanh(x.double())
    e = 0.0
    t = None
    if k["wave_f32"] is not None:
        t = k["wave_f32"].reshape(-1)[:n]
        e = _excess(t, ref, 4 * U32 * ref.abs() + 1e-45)
    if k["wave_i16"] is not None:
        t = torch.tanh(x.float()) if t is None else t
        want = (t.float() * 32768.0).to(torch.int32).to(torch.int16)
        if not torch.equal(k["wave_i16"].reshape(-1)[:n], want):
            e = math.inf
    return e


def check_stft_magnitude(a, k):
    """The hi/lo magnitude operand bit for bit (one IEEE op per step, as the spec); log_mag within 1 ulp of the fp64 log;
    energy: ((ceil(bins / 32) + 6) / 2 + 1) u relative."""
    Fq, bins = a["Fq"], a["bins"]
    re, im = Fq[:, :bins].float(), Fq[:, bins:2 * bins].float()
    m = torch.sqrt((re * re + im * im).double()).float()
    e = 0.0
    if k["mag_op"] is not None:
        want = a["mag_op"].clone()
        S._store_bf16(want, m, a["split_off"])
        e = max(e, 0.0 if torch.equal(_bits(k["mag_op"]), _bits(want)) else math.inf)
    if k["log_mag"] is not None:
        ref = torch.log(torch.clamp(m.double(), min=torch.tensor(a["floor"], dtype=torch.float32).item()))
        e = max(e, _excess(k["log_mag"].reshape(ref.shape), ref, _ulp32(ref)))
    if k["energy"] is not None:
        ref = m.double().pow(2).sum(1).sqrt()
        e = max(e, _excess(k["energy"].reshape(-1), ref, ((math.ceil(bins / 32) + 6) / 2 + 1) * U32 * ref + 1e-45))
    return e


def _ulp32(r):
    return ulp32(r.cpu()).to(r.device)


def check_log_clamp(a, k):
    ref = torch.log(torch.clamp(a["x"].double(), min=torch.tensor(a["floor"], dtype=torch.float32).item()))
    got = k["y"].reshape(ref.shape).double()
    fin = torch.isfinite(ref)
    e = _excess(got[fin], ref[fin], _ulp32(ref[fin]))
    return e if bool((got[~fin] == ref[~fin]).all()) else math.inf


CHECKS = {"conv_gemm": check_conv_gemm, "attention": check_attention, "attention_wide": check_attention_wide,
          "rel_attention": check_rel_attention, "groupnorm_stats": check_groupnorm_stats,
          "groupnorm": check_groupnorm, "layernorm": check_layernorm, "rmsnorm": check_rmsnorm,
          "softmax_rows": check_softmax_rows, "timestep_embedding": check_timestep_embedding,
          "linear_f32": check_linear_f32, "convt_gather": check_convt_gather, "tanh_to_i16": check_tanh_to_i16,
          "stft_magnitude": check_stft_magnitude, "log_clamp": check_log_clamp}
# bit for bit: the statement itself, evaluated on the snapshot
EXACT = ("gather_rows", "cast_act", "transpose_bf16", "stft_frames") + LATENT_STEPS
assert set(CHECKS) | set(EXACT) == set(SPECS)


def _shape(entry, a):
    if entry == "conv_gemm":
        return f"{a['NB']}x{a['H']}x{a['W']} K={a['weight'].shape[1]} N={a['weight'].shape[0]}"
    if entry == "attention_wide":
        return f"{a['batch']}x{a['L']}x{a['dim']}"
    if entry == "attention":
        return f"{a['batch']}x{a['heads']} {a['Lq']}x{a['Lk']}" + (" hi/lo" if a["nsplit"] == 2 else "")
    regs = [r for _, rs, _ in REGIONS[entry](a) for r in rs]
    return "x".join(map(str, regs[0].shape)) if regs else "-"


def _work(entry, a):
    if entry in LATENT_STEPS:
        return a["B"] * a["Cc"] * a["HW"]
    if entry == "cast_act":
        Cc = a["x"].shape[-1] if a["Cc"] is None else a["Cc"]
        return a["NB"] * a["H"] * a["W"] * (4 if a["upsample2x"] else 1) * Cc // 4
    return 0


def _tags(entry, a, launches):
    t = set()
    if entry == "conv_gemm":
        if a["act"] in (L.ACT_GEGLU, L.ACT_GEGLU_TANH):
            t.add("geglu")
        if a["gn_stats"] is not None:      # the after-pass is a second launch (tng_conv_gemm: launch_col_stats)
            t.add("stats-after" if launches == 2 else "stats-fused")
    return frozenset(t)


# ---------------------------------------------------------------------------------------------------- the audit
class Audit:
    def __init__(self, only=None):
        self.only = None if only is None else set(only)
        self.records: list = []
        self.calls = defaultdict(int)        # every wrapped call, audited or passed through
        self.on_device = False

    # one audited call -------------------------------------------------------------------------------------------
    def run(self, entry, orig, args, kwargs):
        self.calls[entry] += 1
        if self.only is not None and entry not in self.only:
            return orig(*args, **kwargs)
        bound = inspect.signature(SPECS[entry]).bind(*args, **kwargs)
        bound.apply_defaults()
        a = dict(bound.arguments)
        a.setdefault("_", {})
        regions = REGIONS[entry](a)
        out_names = {n for n, _, _ in regions}
        stores = {}
        for _, rs, _ in regions:
            for r in rs:
                stores.setdefault(_skey(r), _Storage(r))
        for _, rs, reads in regions:
            for r in rs:
                s = stores[_skey(r)]
                _mark(s.region, r)
                if reads:
                    _mark(s.read, r)
        for n, v in a.items():              # inputs aliased to an output storage (res = out_f32, prev = sample, ...)
            if n not in out_names:
                for t in _read_extents(v):
                    s = stores.get(_skey(t))
                    if s is not None and t.dtype == s.live.dtype:
                        _mark(s.read, t)
        for s in stores.values():           # poison what the kernel must write and does not read
            poison = s.region & ~s.read
            if s.live.dtype.is_floating_point:
                s.live[poison] = float("nan")
            else:
                s.live[poison] = I16_POISON
        dev = next((t.device for v in a.values() for t in _tensors(v)), torch.device("cpu"))
        self.on_device = self.on_device or dev.type == "cuda"
        n0 = L.launch_count() if dev.type == "cuda" else 0
        family = entry
        if dev.type == "cuda":
            prof_was = L.PROF.enabled
            if not prof_was:
                L.PROF.start()
            try:
                result = orig(*args, **kwargs)
            finally:                        # a failed call must not leave the profiler on for the next one
                fams = L.PROF.stop() if not prof_was else {}
            if not prof_was:
                family = next(iter(fams)) if len(fams) == 1 else entry
            torch.cuda.synchronize()
        else:
            result = orig(*args, **kwargs)
        launches = (L.launch_count() - n0) if dev.type == "cuda" else 1
        index = len(self.records)
        where = f"launch #{index} {entry} [{family}] {_shape(entry, a)}"
        for s in stores.values():           # untouched bytes
            keep = ~s.region
            if not torch.equal(_bits(s.live)[keep], _bits(s.snap)[keep]):
                bad = int((_bits(s.live)[keep] != _bits(s.snap)[keep]).sum())
                raise AuditFailure(f"{where}: {bad} element(s) outside the contract region changed")
        ref = {n: _remap_arg(v, stores) for n, v in a.items()}
        if entry in EXACT:
            SPECS[entry](**{n: v for n, v in ref.items() if n != "_"})
            e = 0.0
            for s in stores.values():
                if not torch.equal(_bits(s.live), _bits(s.snap)):
                    bad = int((_bits(s.live) != _bits(s.snap)).sum())
                    raise AuditFailure(f"{where}: {bad} element(s) differ from the statement (bit for bit)")
        else:
            e = CHECKS[entry](ref, a)
        if not e <= 1.0:
            raise AuditFailure(f"{where}: worst excess {e:.3g} over the contract bound")
        self.records.append(Record(index, entry, family, _shape(entry, a), e, launches, _tags(entry, a, launches),
                                   _work(entry, a)))
        return result

    # summaries ---------------------------------------------------------------------------------------------------
    def families(self):
        out = {}
        for r in self.records:
            n, w = out.get((r.entry, r.family), (0, 0.0))
            out[(r.entry, r.family)] = (n + 1, max(w, r.excess))
        return out

    def audited(self):
        return {r.entry for r in self.records}

    def tags(self):
        return set().union(*(r.tags for r in self.records)) if self.records else set()

    def table(self, title=""):
        lines = [f"launch audit {title}: {len(self.records)} launches checked"]
        for (entry, fam), (n, w) in sorted(self.families().items()):
            lines.append(f"  {entry:<20s} {fam:<22s} {n:6d} launches  worst excess {w:.3f}")
        return "\n".join(lines)


def install_audit(monkeypatch, only=None) -> Audit:
    """Wrap every kernel wrapper of tango_b200.lib (whatever it currently is: the library binding, or a spec statement
    under install_spec_backend) in the audit, under pytest's monkeypatch. `only`: entry points to check; the other
    launches pass through."""
    audit = Audit(only)
    for name in SPECS:
        orig = getattr(L, name)

        def wrapped(*args, _name=name, _orig=orig, **kwargs):
            return audit.run(_name, _orig, args, kwargs)

        monkeypatch.setattr(L, name, wrapped)
    return audit
