"""Executable statement of what `tng_conv_gemm` computes from its descriptor (TEST INFRASTRUCTURE ONLY).

include/tango_b200.h describes the operator in prose; this is the same contract in a few lines of torch on the CPU, so
that the host-side packing logic (tango_b200/ops.py: weight layout, k-groups, parity views, hi/lo splitting, GEGLU row
interleave) can be checked against torch convolutions without a GPU. It is never imported by the package.

For output pixel (n, h, w) of the (NB, H, W) grid and output column j:
    acc[row, j] = sum over k-groups g, kk in [0, 64 * nkb):  A_g[row, kk] * B[j, b_k0 + kk]
    A_g[row, kk] = view[g.view] at (n, h + dh, w + dw, a_c0 + kk), ZERO outside the view's (NB, H, W, C) extent
    B[j, k] = weight[j, k], ZERO for k >= Ktot (what the TMA out-of-bounds fill provides)
    y = (acc + bias[j] + rowvec[n, j] + res[row, j]) * alpha (+ previous out_f32 if accumulate);  out_f32 = y
    out_bf16 = act(y) (SiLU / leaky-ReLU), or for GEGLU out[:, tn*BN/2 + i] = y[:, tn*BN + i] * gelu(y[:, tn*BN + BN/2 + i]);
    in split mode the bf16 rounding residual goes to column offset split_off.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

ACT_NONE, ACT_SILU, ACT_LRELU, ACT_GEGLU, ACT_GEGLU_TANH = 0, 1, 2, 3, 4
BK = 64


def _gather_view(v, n_idx, h_idx, w_idx, c0, nk):
    """[rows, nk] fp64 values of view v at (n, h, w, c0 + kk) with zero fill outside the view extent."""
    flat = v.t.reshape(-1).double()
    ok = (h_idx >= 0) & (h_idx < v.H) & (w_idx >= 0) & (w_idx < v.W) & (n_idx >= 0) & (n_idx < v.NB)
    base = v.off + n_idx.clamp(0, v.NB - 1) * v.s_n + h_idx.clamp(0, v.H - 1) * v.s_h + w_idx.clamp(0, v.W - 1) * v.s_w
    c = c0 + torch.arange(nk, device=flat.device)
    c_ok = c < v.C
    idx = base[:, None] + c.clamp(max=max(v.C - 1, 0))[None, :]
    vals = flat[idx.clamp(0, flat.numel() - 1)]
    return vals * (ok[:, None] & c_ok[None, :])


def spec_conv_gemm(views, groups, weight, W, H, NB, *, bias=None, rowvec=None, res=None, alpha=1.0, accumulate=False,
                   out_f32=None, out_bf16=None, act=ACT_NONE, act_param=0.0, split_off=0, block_n=0, rowvec_ld=0,
                   gn_stats=None, stats_hw=0, **_):
    rows = NB * H * W
    dev = weight.device
    r = torch.arange(rows, device=dev)
    n_idx, h_idx, w_idx = r // (H * W), (r // W) % H, r % W
    Ncols, Ktot = weight.shape
    wd = weight.double()
    acc = torch.zeros(rows, Ncols, dtype=torch.float64, device=dev)
    for (vi, a_c0, dw, dh, b_k0, nkb) in groups:
        nk = nkb * BK
        a = _gather_view(views[vi], n_idx, h_idx + dh, w_idx + dw, a_c0, nk)
        b = torch.zeros(Ncols, nk, dtype=torch.float64, device=dev)
        kmax = max(0, min(nk, Ktot - b_k0))
        b[:, :kmax] = wd[:, b_k0:b_k0 + kmax]
        acc += a @ b.t()
    y = acc
    if bias is not None:
        y = y + bias.double()[None, :]
    if rowvec is not None:
        ld = rowvec_ld or Ncols
        nimg = int(n_idx.max()) + 1
        rv = rowvec.as_strided((nimg, Ncols), (ld, 1)).double()     # pointer + leading dimension, as the ABI sees it
        y = y + rv[n_idx]
    if res is not None:
        y = y + res.double()[:, :Ncols]
    y = y * alpha
    if out_f32 is not None:
        if accumulate:        # the accumulated value is also what the bf16 output (if any) is derived from
            y = y + out_f32[:, :Ncols].double()
        out_f32[:, :Ncols] = y.float()
    if gn_stats is not None:   # per-(image, channel) sums of the stored value are ADDED to the accumulators: the fp32
        # output, else the (plain) bf16 one
        yi = (y.float() if out_f32 is not None else y.float().bfloat16()).double().view(rows // stats_hw, stats_hw, Ncols)
        gn_stats[..., 0] += yi.sum(1)
        gn_stats[..., 1] += (yi * yi).sum(1)
    if out_bf16 is not None:
        z = y.float()
        if act == ACT_SILU:
            z = F.silu(z)
        elif act == ACT_LRELU:
            z = F.leaky_relu(z, act_param)
        elif act in (ACT_GEGLU, ACT_GEGLU_TANH):
            bn = block_n
            assert bn in (128, 256) and Ncols % bn == 0
            assert alpha == 1.0 and res is None and rowvec is None   # tng_conv_gemm: TNG_EINVAL otherwise
            t = z.view(rows, Ncols // bn, bn)
            gate = F.gelu(t[..., bn // 2:], approximate="tanh" if act == ACT_GEGLU_TANH else "none")
            z = (t[..., :bn // 2] * gate).reshape(rows, Ncols // 2)
        hi = z.to(torch.bfloat16)
        out_bf16[:, :z.shape[1]] = hi
        if split_off > 0:
            out_bf16[:, split_off:split_off + z.shape[1]] = (z - hi.float()).to(torch.bfloat16)


# ---------------------------------------------------------------------------------------------------------------------
# The other entry points of include/tango_b200.h, same purpose: torch-CPU statements of the contracts, installed by
# `install_spec_backend` to run the package's host orchestration (weight packing, buffer plumbing, operator sequencing
# of unet.py / t5.py, the sampling and editing loops) without a GPU. Every function mirrors the signature of its
# tango_b200.lib wrapper.
def _store_bf16(y, z, split_off):
    hi = z.to(torch.bfloat16)
    n = z.shape[1]
    y[:, :n] = hi
    if split_off > 0:
        y[:, split_off:split_off + n] = (z - hi.float()).to(torch.bfloat16)


def _act(z, act, act_param=0.0):
    if act == ACT_SILU:
        return F.silu(z)
    if act == ACT_LRELU:
        return F.leaky_relu(z, act_param)
    return z


def spec_groupnorm_stats(x, NB, HW, stats):
    xi = x.double().view(NB, HW, x.shape[-1])
    stats[..., 0] += xi.sum(1)
    stats[..., 1] += (xi * xi).sum(1)


def spec_groupnorm(x0, st0, x1, st1, NB, HW, groups, gamma, beta, eps, act, y, *, split_off=0, raw=None, raw_split_off=0):
    """Normalisation with the group mean / variance taken from the per-channel accumulators (sum, sum of squares), as
    the kernel does: mean = S / n, var = Q / n - mean^2 over the channels of the group in the concat [x0 | x1]."""
    x = x0.float() if x1 is None else torch.cat([x0.float(), x1.float()], dim=-1)
    C_ = x.shape[1]
    st = st0 if x1 is None else torch.cat([st0, st1], dim=1)            # [NB, C, 2]
    cpg = C_ // groups
    gs = st.view(NB, groups, cpg, 2).sum(2)
    n = float(HW * cpg)
    mean = gs[..., 0] / n
    var = (gs[..., 1] / n - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + eps)
    mean_c = mean.float().repeat_interleave(cpg, 1)[:, None, :]
    rstd_c = rstd.float().repeat_interleave(cpg, 1)[:, None, :]
    z = ((x.view(NB, HW, C_) - mean_c) * rstd_c * gamma + beta).reshape(NB * HW, C_)
    _store_bf16(y, _act(z, act), split_off)
    if raw is not None:
        _store_bf16(raw, x, raw_split_off)


def spec_layernorm(x, gamma, beta, eps, y, *, split_off=0):
    _store_bf16(y, F.layer_norm(x.float(), (x.shape[1],), gamma, beta, eps), split_off)


def spec_rmsnorm(x, gamma, eps, y=None, *, split_off=0, y_f32=None):
    z = gamma * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))
    if y is not None:
        _store_bf16(y, z, split_off)
    if y_f32 is not None:
        y_f32.copy_(z)


def spec_gather_rows(table, ids, out):
    out.copy_(table[ids])


def spec_cast_act(x, NB, H, W, y, *, Cc=None, upsample2x=False, act=ACT_NONE, act_param=0.0, split_off=0):
    Cc = x.shape[-1] if Cc is None else Cc
    z = x[:, :Cc].float()
    if upsample2x:
        z = z.view(NB, H, W, Cc).repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(NB * 4 * H * W, Cc)
    _store_bf16(y, _act(z, act, act_param), split_off)


def _heads(t, col0, lo_off, nsplit, B, L_, heads):
    v = t[:, col0:col0 + heads * 64].float()
    if nsplit == 2:
        v = v + t[:, col0 + lo_off:col0 + lo_off + heads * 64].float()
    return v.view(B, L_, heads, 64).transpose(1, 2)


def spec_attention(q, k, v, out, *, batch, heads, Lq, Lk, scale, q_col0=0, k_col0=0, v_col0=0, kbias=None, nsplit=1,
                   q_lo_off=0, k_lo_off=0, v_lo_off=0, split_off=0):
    qh = _heads(q, q_col0, q_lo_off, nsplit, batch, Lq, heads)
    kh = _heads(k, k_col0, k_lo_off, nsplit, batch, Lk, heads)
    vh = _heads(v, v_col0, v_lo_off, nsplit, batch, Lk, heads)
    s = qh @ kh.transpose(-1, -2) * scale
    if kbias is not None:
        s = s + kbias.view(batch, 1, 1, Lk)
    o = (s.softmax(-1) @ vh).transpose(1, 2).reshape(batch * Lq, heads * 64)
    _store_bf16(out, o, split_off)


def spec_attention_wide(q, k, v, out, *, batch, L, dim, scale, q_col0=0, k_col0=0, v_col0=0):
    qh, kh, vh = (t[:, c:c + dim].float().view(batch, L, dim) for t, c in ((q, q_col0), (k, k_col0), (v, v_col0)))
    o = (qh @ kh.transpose(1, 2) * scale).softmax(-1) @ vh
    out[:, :dim] = o.reshape(batch * L, dim).to(torch.bfloat16)


def spec_rel_attention(qkv, relbias, kbias, out, *, batch, heads, L, q_col0, k_col0, v_col0, split_off=0):
    inner = heads * 64
    q, k, v = (qkv[:, c:c + inner].view(batch, L, heads, 64).transpose(1, 2) for c in (q_col0, k_col0, v_col0))
    pos = torch.arange(L)
    bias = relbias[:, (pos[None, :] - pos[:, None]) + L - 1][None]
    if kbias is not None:
        bias = bias + kbias.view(batch, 1, 1, L)
    o = ((q @ k.transpose(-1, -2) + bias).softmax(-1) @ v).transpose(1, 2).reshape(batch * L, inner)
    _store_bf16(out, o, split_off)


def spec_timestep_embedding(t, dim, flip_sin_to_cos, freq_shift, out):
    import math
    half = dim // 2
    e = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32) / (half - freq_shift))
    a = t.float()[:, None] * e[None, :]
    out.copy_(torch.cat([torch.cos(a), torch.sin(a)] if flip_sin_to_cos else [torch.sin(a), torch.cos(a)], dim=-1))


def spec_linear_f32(x, w, b, y, *, pre_act=ACT_NONE, post_act=ACT_NONE):
    y.copy_(_act(F.linear(_act(x.float(), pre_act), w, b), post_act))


def spec_softmax_rows(x, scale, y, *, L=None, split_off=0):
    L_ = x.shape[1] if L is None else L
    _store_bf16(y, torch.softmax(x[:, :L_].float() * scale, dim=-1), split_off)


def spec_transpose_bf16(x, B, R, Cc, y):
    """x: bf16 [B*R, >=Cc] -> y: bf16 [B*Cc, >=R], each of the B [R, Cc] blocks transposed."""
    y[:B * Cc, :R] = x[:B * R, :Cc].reshape(B, R, Cc).transpose(1, 2).reshape(B * Cc, R)


def spec_convt_gather(Y, B, Lin, ktaps, Cout, stride, pad, Lout, bias, y):
    """ConvTranspose1d overlap-add: y[b, l, :] = bias + sum over (q, t) with q*stride + t - pad == l of Y[b, q, t, :]."""
    Yv = Y.reshape(B, Lin, ktaps, Cout).double()
    out = torch.zeros(B, Lout, Cout, dtype=torch.float64, device=Y.device)
    for t in range(ktaps):
        l = torch.arange(Lin, device=Y.device) * stride + t - pad
        ok = (l >= 0) & (l < Lout)
        out[:, l[ok], :] += Yv[:, ok, t, :]
    if bias is not None:
        out = out + bias.double()
    y.reshape(B, Lout, Cout).copy_(out.float())


def spec_tanh_to_i16(x, n, ld_x, wave_f32, wave_i16):
    t = torch.tanh(x.reshape(-1)[: n * ld_x: ld_x].float())
    if wave_f32 is not None:
        wave_f32.reshape(-1)[:n] = t
    if wave_i16 is not None:   # float32 product, truncation toward zero, wrap to int16 (numpy astype semantics)
        wave_i16.reshape(-1)[:n] = (t * 32768.0).to(torch.int32).to(torch.int16)


# The latent updates (tng_sched_step, tng_dpm_step, tng_latent_blend): one op per kernel op, same association.
# model_out: channels-last rows [(2)B*HW, >=Cc] fp32; sample / noise / prev / history: NCHW fp32; next_in: channels-last
# bf16 rows [(2)B*HW, ld_in].
def _guided_output(model_out, cfg, guidance, *, B, Cc, HW):
    """The model output as [B, Cc, HW]: u + guidance * (t - u) under CFG (uncond rows first)."""
    mo = model_out[:, :Cc].float()
    if cfg:
        u, t = mo[:B * HW].reshape(B, HW, Cc), mo[B * HW:2 * B * HW].reshape(B, HW, Cc)
        v = u + guidance * (t - u)
    else:
        v = mo[:B * HW].reshape(B, HW, Cc)
    return v.transpose(1, 2)


def _pack_next_in(next_in, x, cfg, split_off, *, B, Cc, HW):
    """The new latent x [B, Cc, HW] as the next UNet input: once per CFG half, hi/lo split at split_off."""
    if next_in is not None:
        rows = x.transpose(1, 2).reshape(B * HW, Cc)
        for r in range(2 if cfg else 1):
            _store_bf16(next_in[r * B * HW:(r + 1) * B * HW], rows, split_off)


def spec_sched_step(model_out, cfg, guidance, sample, noise, coef, prev, next_in, *, B, Cc, HW, split_off=0):
    """CFG combine + scheduler update (coefficient row `coef`, see schedulers.py) + packing of the next UNet input."""
    c = [coef.reshape(-1)[i] for i in range(10)]
    s = sample.reshape(B, Cc, HW).float()
    out = s
    if model_out is not None:
        v = _guided_output(model_out, cfg, guidance, B=B, Cc=Cc, HW=HW)
        x0 = (c[0] * s + c[1] * v) / c[9]
        if float(c[8]) > 0:
            x0 = x0.clamp(-float(c[8]), float(c[8]))
        out = c[2] * x0 + c[3] * s
        if float(c[7]) != 0:
            out = out + c[7] * (c[5] * s + c[6] * v)
        if noise is not None and float(c[4]) != 0:
            out = out + c[4] * noise.reshape(B, Cc, HW)
    if prev is not None:
        prev.reshape(B, Cc, HW).copy_(out)
    _pack_next_in(next_in, out, cfg, split_off, B=B, Cc=Cc, HW=HW)


def spec_dpm_step(model_out, cfg, guidance, sample, coef, order, m0, m1, m2, prev, next_in, *, B, Cc, HW, split_off=0):
    """CFG combine + DPM-Solver(++) update of `order` from the history slots m0 (written) / m1 / m2 + packing."""
    c = [coef.reshape(-1)[i] for i in range(11)]
    s = sample.reshape(B, Cc, HW).float()
    v = _guided_output(model_out, cfg, guidance, B=B, Cc=Cc, HW=HW)
    x0 = (c[0] * s + c[1] * v) / c[2]
    m0.reshape(B, Cc, HW).copy_(x0)
    x = c[3] * s - c[4] * x0
    if order == 2:
        x = x + c[5] * (c[7] * (x0 - m1.reshape(B, Cc, HW)))
    elif order == 3:
        p1, p2 = m1.reshape(B, Cc, HW), m2.reshape(B, Cc, HW)
        d1_0, d1_1 = c[7] * (x0 - p1), c[8] * (p1 - p2)
        dd = d1_0 - d1_1
        x = (x + c[5] * (d1_0 + c[9] * dd)) - c[6] * (c[10] * dd)
    if prev is not None:
        prev.reshape(B, Cc, HW).copy_(x)
    _pack_next_in(next_in, x, cfg, split_off, B=B, Cc=Cc, HW=HW)


def spec_latent_blend(x0, noise, mask, coef, sample, next_in=None, *, B, Cc, HW, cfg=False, split_off=0):
    """add_noise(x0, noise) (mask None) or add_noise(x0, noise) * m + sample * (1 - m), written to sample + packing."""
    c = coef.reshape(-1)
    p = c[0] * x0.reshape(B, Cc, HW).float()
    if noise is not None:
        p = p + c[1] * noise.reshape(B, Cc, HW).float()
    if mask is not None:
        m = mask.reshape(-1, 1, HW)
        p = (p * m) + (sample.reshape(B, Cc, HW) * (1 - m))
    sample.reshape(B, Cc, HW).copy_(p)
    _pack_next_in(next_in, p, cfg, split_off, B=B, Cc=Cc, HW=HW)


def spec_stft_frames(y, pad, hi, lo):
    """Reflect padding (no edge repeat) by `pad` on both sides, bf16 hi / lo planes, zero beyond T + 2 pad."""
    B, T = y.shape
    z = torch.zeros(B, hi.shape[1], device=y.device)
    z[:, :T + 2 * pad] = F.pad(y.float().view(B, 1, T), (pad, pad), mode="reflect").view(B, -1)
    h = z.to(torch.bfloat16)
    hi.copy_(h)
    lo.copy_((z - h.float()).to(torch.bfloat16))


def spec_stft_magnitude(Fq, bins, mag_op, split_off, log_mag, energy, floor=1e-5):
    re, im = Fq[:, :bins].float(), Fq[:, bins:2 * bins].float()
    # IEEE sqrt of the fp32 sum (torch's vectorised fp32 sqrt on the CPU is not always correctly rounded; the fp64 root
    # of an fp32 value rounds to the correctly rounded fp32 root)
    m = torch.sqrt((re * re + im * im).double()).float()
    if mag_op is not None:
        _store_bf16(mag_op, m, split_off)
    if log_mag is not None:
        log_mag.copy_(torch.log(torch.clamp(m, min=floor)))
    if energy is not None:
        energy.copy_(torch.norm(m, dim=1))


def spec_log_clamp(x, y, floor=1e-5):
    y.copy_(torch.log(torch.clamp(x.float(), min=floor)))


SPEC = {"attention_wide": spec_attention_wide, "stft_frames": spec_stft_frames, "stft_magnitude": spec_stft_magnitude, "log_clamp": spec_log_clamp,
        "softmax_rows": spec_softmax_rows, "transpose_bf16": spec_transpose_bf16, "convt_gather": spec_convt_gather,
        "tanh_to_i16": spec_tanh_to_i16, "sched_step": spec_sched_step, "dpm_step": spec_dpm_step,
        "latent_blend": spec_latent_blend, "conv_gemm": spec_conv_gemm, "groupnorm": spec_groupnorm, "groupnorm_stats": spec_groupnorm_stats, "layernorm": spec_layernorm, "rmsnorm": spec_rmsnorm,
        "gather_rows": spec_gather_rows, "cast_act": spec_cast_act, "attention": spec_attention,
        "rel_attention": spec_rel_attention, "timestep_embedding": spec_timestep_embedding, "linear_f32": spec_linear_f32}


def install_spec_backend(monkeypatch):
    """Run the package's host code on CPU tensors: every kernel wrapper of tango_b200.lib becomes its statement in
    SPEC, and the device checks, the library load and the launch counter become no-ops (under pytest's monkeypatch
    only, so nothing here is a CPU fallback of the product)."""
    from tango_b200 import lib as L
    for name, fn in SPEC.items():
        monkeypatch.setattr(L, name, fn)
    monkeypatch.setattr(L, "require_cuda_device", lambda device: None)
    monkeypatch.setattr(L, "require_cuda", lambda *ts: None)
    monkeypatch.setattr(L, "load", lambda *a, **k: None)
    monkeypatch.setattr(L, "launch_count", lambda: 0)
