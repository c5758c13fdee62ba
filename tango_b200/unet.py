"""UNet2DConditionModel for the Tango hot path, running on the hand-written sm_90a kernels.

Drop-in for diffusers' UNet2DConditionModel as Tango uses it (config JSON, 686-tensor state_dict layout,
`load_config / from_config / load_state_dict / forward(...).sample / .config.in_channels`;
/root/reference/mustango/diffusers/src/diffusers/models/unet_2d_condition.py:520-707, unet_2d_blocks.py,
resnet.py:549-597, transformer_2d.py:214-321, attention.py:276-335, attention_processor.py:263-299).

Layout: activations are channels-last row matrices ([B*H*W, C]); the residual stream is fp32, tensor-core operands
are bf16 (precision="bf16") or bf16 hi/lo pairs (precision="split", ~fp32 accuracy: the parity mode).
Per forward: GroupNorm(+SiLU) -> wgmma implicit-GEMM conv (bias + time-embedding + residual / fused 1x1
shortcut in the epilogue) for the resnets; GroupNorm -> GEMM -> [LayerNorm -> fused-QKV GEMM -> wgmma flash
attention -> out-proj(+residual)] x2 (cross-attention K/V are step-invariant and cached per prompt batch)
-> LayerNorm -> GEGLU GEMM -> GEMM(+residual) -> proj_out(+residual) for the transformers.
"""
from __future__ import annotations

import json
from types import SimpleNamespace
from typing import Dict, List, Optional

import torch

from . import blocks
from . import lib as L
from .blocks import Buffers, Packer, StatsArena
from .ops import PackedConv, run_linear


class UNetOutput(SimpleNamespace):
    pass


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def _heads(cfg) -> List[int]:
    ahd = cfg["attention_head_dim"]
    return list(ahd) if isinstance(ahd, (list, tuple)) else [ahd] * len(cfg["block_out_channels"])


class UNet2DConditionModel:
    """See module docstring. `precision`: "bf16" (perf) or "split" (parity)."""

    SUPPORTED_DOWN = ("CrossAttnDownBlock2D", "DownBlock2D", "CrossAttnDownBlock2DMusic")
    SUPPORTED_UP = ("CrossAttnUpBlock2D", "UpBlock2D", "CrossAttnUpBlock2DMusic")
    # The *Music types are the Mustango variant (SURVEY.md section 8(f).4; D/models/unet_2d_condition_music.py:536-757,
    # unet_2d_blocks.py:603-760,1079-1270,2251-2440): every attention position runs two more Transformer2DModels
    # (`attentions2` on beat features, `attentions3` on chord features) right after the text one.

    def __init__(self, config: dict, precision: str = "bf16"):
        cfg = dict(config)
        for bt in cfg["down_block_types"]:
            if bt not in self.SUPPORTED_DOWN:
                raise NotImplementedError(f"down block type {bt} is not on the Tango path")
        for bt in cfg["up_block_types"]:
            if bt not in self.SUPPORTED_UP:
                raise NotImplementedError(f"up block type {bt} is not on the Tango path")
        if not cfg.get("use_linear_projection", False):
            raise NotImplementedError("use_linear_projection=False is not on the Tango path")
        if any(c % 64 for c in cfg["block_out_channels"]):
            raise NotImplementedError("block_out_channels must be multiples of 64")
        hd = [c // h for c, h in zip(cfg["block_out_channels"], _heads(cfg))]
        if any(d != 64 for d in hd):
            raise NotImplementedError(f"attention head width must be 64 (got {hd})")
        # config fields this implementation does not honour are refused, not ignored (the Tango / Mustango configs
        # all use the values below; unet_2d_condition.py:130-330; upcast_attention is moot: scores / softmax are fp32)
        unsupported = {"norm_num_groups": 32, "act_fn": "silu", "class_embed_type": None, "only_cross_attention": False,
                       "center_input_sample": False, "downsample_padding": 1, "dual_cross_attention": False,
                       "resnet_time_scale_shift": "default", "time_embedding_type": "positional",
                       "num_class_embeds": None, "conv_in_kernel": 3, "conv_out_kernel": 3, "mid_block_scale_factor": 1,
                       "time_cond_proj_dim": None, "timestep_post_act": None, "projection_class_embeddings_input_dim": None}
        for k, want in unsupported.items():
            if k in cfg and cfg[k] != want and not (want is False and not cfg[k]):
                raise NotImplementedError(f"UNet config {k}={cfg[k]!r} is not on the Tango path (supported: {want!r})")
        assert precision in ("bf16", "split")
        self.config = _Cfg(cfg)
        self.precision = precision
        self.split = precision == "split"
        self.s = 2 if self.split else 1
        self.device = torch.device("cpu")
        self.dtype = torch.float32
        self._sd: Optional[Dict[str, torch.Tensor]] = None
        self._packed = False
        self.pack_generation = 0     # bumped whenever the packed weights / scratch buffers are rebuilt
        self._bufs: Optional[Buffers] = None
        self._cond = None

    # ----------------------------------------------------------------------------------------- diffusers-style API
    @staticmethod
    def load_config(path: str, **_kw) -> dict:
        with open(path) as f:
            return json.load(f)

    @classmethod
    def from_config(cls, config: dict, precision: str = "bf16", **_kw) -> "UNet2DConditionModel":
        return cls({k: v for k, v in config.items() if not k.startswith("_")}, precision=precision)

    def to(self, device=None, *_a, **_k):
        if device is not None and not isinstance(device, torch.dtype):
            device = torch.device(device)
            if device != self.device:
                self.device = device
                self._packed = False
        return self

    def eval(self):
        return self

    def parameters_shapes(self):
        from .synth import unet_param_shapes
        return unet_param_shapes(self.config)

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        want = self.parameters_shapes()
        missing = [k for k in want if k not in sd]
        unexpected = [k for k in sd if k not in want]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:5]}..., unexpected {unexpected[:5]}...")
        for k, shp in want.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise RuntimeError(f"size mismatch for {k}: {tuple(sd[k].shape)} vs {tuple(shp)}")
        self._sd = {k: v.detach() for k, v in sd.items() if k in want}
        self._packed = False
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    # ----------------------------------------------------------------------------------------- weight packing
    def _pack(self):
        if self._packed:
            return
        if self._sd is None:
            raise L.TangoB200Error("UNet2DConditionModel has no weights: call load_state_dict first")
        L.require_cuda_device(self.device)
        L.load()
        sd, dev, sp = self._sd, self.device, self.split
        cfg = self.config
        boc = cfg["block_out_channels"]
        P: Dict[str, object] = {}
        pk = Packer(sd, dev, sp)
        f32, conv = pk.f32, pk.conv

        def resnet(p):
            r = pk.resnet(p, "conv_shortcut", cfg.get("norm_eps", 1e-5))
            r.temb_w, r.temb_b = sd[p + ".time_emb_proj.weight"].float(), sd[p + ".time_emb_proj.bias"].float()
            return r

        def transformer(p, heads):
            t = SimpleNamespace()
            t.heads = heads
            t.nw, t.nb = f32(p + ".norm.weight"), f32(p + ".norm.bias")
            t.proj_in, t.proj_out = conv(p + ".proj_in"), conv(p + ".proj_out")
            b = p + ".transformer_blocks.0"
            for i in (1, 2, 3):
                setattr(t, f"ln{i}w", f32(f"{b}.norm{i}.weight"))
                setattr(t, f"ln{i}b", f32(f"{b}.norm{i}.bias"))
            wqkv = torch.cat([sd[f"{b}.attn1.to_q.weight"], sd[f"{b}.attn1.to_k.weight"], sd[f"{b}.attn1.to_v.weight"]], 0)
            t.qkv = PackedConv(wqkv, None, split=sp, device=dev)
            t.out1 = conv(f"{b}.attn1.to_out.0")
            t.q2 = conv(f"{b}.attn2.to_q")
            t.kv2 = PackedConv(torch.cat([sd[f"{b}.attn2.to_k.weight"], sd[f"{b}.attn2.to_v.weight"]], 0), None,
                               split=sp, device=dev)
            t.out2 = conv(f"{b}.attn2.to_out.0")
            cdim = t.proj_in.cout
            inner8 = 8 * cdim
            t.ff1 = conv(f"{b}.ff.net.0.proj", geglu_bn=256 if inner8 % 256 == 0 else 128)
            t.ff2 = conv(f"{b}.ff.net.2")
            t.C = cdim
            return t

        heads = _heads(cfg)
        lpb = cfg["layers_per_block"]
        P["conv_in"] = conv("conv_in")
        P["down"] = []
        for i, bt in enumerate(cfg["down_block_types"]):
            blk = SimpleNamespace(resnets=[], attns=[], down=None)
            for j in range(lpb):
                blk.resnets.append(resnet(f"down_blocks.{i}.resnets.{j}"))
                if bt in ("CrossAttnDownBlock2D", "CrossAttnDownBlock2DMusic"):
                    blk.attns.append(transformer(f"down_blocks.{i}.attentions.{j}", heads[i]))
                    blk.attns[-1].extra = [transformer(f"down_blocks.{i}.attentions{n}.{j}", heads[i])
                                           for n in ((2, 3) if bt.endswith("Music") else ())]
            if i != len(boc) - 1:
                blk.down = conv(f"down_blocks.{i}.downsamplers.0.conv", stride=2)
            P["down"].append(blk)
        P["mid"] = SimpleNamespace(r0=resnet("mid_block.resnets.0"), attn=transformer("mid_block.attentions.0", heads[-1]),
                                   r1=resnet("mid_block.resnets.1"))
        mid_music = cfg.get("mid_block_type", "UNetMidBlock2DCrossAttn") == "UNetMidBlock2DCrossAttnMusic"
        P["mid"].attn.extra = [transformer(f"mid_block.attentions{n}.0", heads[-1]) for n in ((2, 3) if mid_music else ())]
        rheads = list(reversed(heads))
        P["up"] = []
        for i, bt in enumerate(cfg["up_block_types"]):
            blk = SimpleNamespace(resnets=[], attns=[], up=None)
            for j in range(lpb + 1):
                blk.resnets.append(resnet(f"up_blocks.{i}.resnets.{j}"))
                if bt in ("CrossAttnUpBlock2D", "CrossAttnUpBlock2DMusic"):
                    blk.attns.append(transformer(f"up_blocks.{i}.attentions.{j}", rheads[i]))
                    blk.attns[-1].extra = [transformer(f"up_blocks.{i}.attentions{n}.{j}", rheads[i])
                                           for n in ((2, 3) if bt.endswith("Music") else ())]
            if i != len(boc) - 1:
                blk.up = conv(f"up_blocks.{i}.upsamplers.0.conv")
            P["up"].append(blk)
        P["norm_out"] = (f32("conv_norm_out.weight"), f32("conv_norm_out.bias"))
        P["conv_out"] = conv("conv_out")
        # time embedding: linear_1 / linear_2 and ALL resnet time_emb_proj layers concatenated into one matrix
        P["te1"] = (f32("time_embedding.linear_1.weight"), f32("time_embedding.linear_1.bias"))
        P["te2"] = (f32("time_embedding.linear_2.weight"), f32("time_embedding.linear_2.bias"))
        res_all = [r for b in P["down"] for r in b.resnets] + [P["mid"].r0, P["mid"].r1] + [r for b in P["up"] for r in b.resnets]
        off = 0
        for r in res_all:
            r.temb_off = off
            off += r.cout
        P["temb_total"] = off
        P["temb_w"] = torch.cat([r.temb_w for r in res_all], 0).contiguous().to(dev)
        P["temb_b"] = torch.cat([r.temb_b for r in res_all], 0).contiguous().to(dev)
        P["transformers"] = [t for b in P["down"] for t in b.attns] + [P["mid"].attn] + [t for b in P["up"] for t in b.attns]
        P["n_extra"] = max((len(t.extra) for t in P["transformers"]), default=0)
        tr_all = list(P["transformers"]) + [x for t in P["transformers"] for x in t.extra]
        P["stat_channels"] = blocks.stat_channels(P["conv_in"], res_all, tr_all,
                                                  [b.down for b in P["down"]] + [b.up for b in P["up"]])
        self.P = P
        self._bufs = Buffers(dev)
        self._arenas: Dict[int, StatsArena] = {}
        self._cond = None
        self.pack_generation += 1
        self._packed = True

    # ----------------------------------------------------------------------------------------- building blocks
    def time_embedding_table(self, timesteps: torch.Tensor) -> torch.Tensor:
        """[n] timesteps -> [n, temb_total] fp32: every resnet's Linear(SiLU(TimestepEmbedding(t))) in one table
        (embeddings.py:22-62,200-212; resnet.py:572-573). Exact fp32 SIMT kernels; batch- and data-independent."""
        self._pack()
        P, cfg = self.P, self.config
        n = timesteps.numel()
        t = timesteps.to(self.device, torch.float32).contiguous()
        c0 = cfg["block_out_channels"][0]
        e0 = torch.empty(n, c0, device=self.device)
        L.timestep_embedding(t, c0, cfg.get("flip_sin_to_cos", True), float(cfg.get("freq_shift", 0)), e0)
        e1 = torch.empty(n, 4 * c0, device=self.device)
        L.linear_f32(e0, P["te1"][0], P["te1"][1], e1, post_act=L.ACT_SILU)
        e2 = torch.empty(n, 4 * c0, device=self.device)
        L.linear_f32(e1, P["te2"][0], P["te2"][1], e2)
        out = torch.empty(n, P["temb_total"], device=self.device)
        L.linear_f32(e2, P["temb_w"], P["temb_b"], out, pre_act=L.ACT_SILU)
        return out

    def set_conditioning(self, encoder_hidden_states: torch.Tensor, encoder_attention_mask: Optional[torch.Tensor],
                         extra_streams=()):
        """Project the (frozen, step-invariant) text states to K/V for all 16 cross-attention layers once
        (attention_processor.py:279-284) and turn the mask into the additive bias of unet_2d_condition.py:575-579.
        `extra_streams`: ((features [Bu, L, D], mask or None), ...) for the Mustango blocks — beats, then chords."""
        self._pack()
        if len(extra_streams) != self.P["n_extra"]:
            raise L.TangoB200Error(f"this UNet needs {self.P['n_extra']} extra conditioning streams, got {len(extra_streams)}")
        ehs = encoder_hidden_states.to(self.device, torch.float32, non_blocking=True).contiguous()
        Bu, Lk, D = ehs.shape
        s = self.s
        # persistent buffers (same addresses on every call with the same shapes -> a captured CUDA graph stays valid)
        eb = self._bufs.get("cond_ehs", (Bu * Lk, D * s), torch.bfloat16)
        L.cast_act(ehs.view(Bu * Lk, D), 1, 1, Bu * Lk, eb, split_off=D if self.split else 0)
        kvs = []
        for i, t in enumerate(self.P["transformers"]):
            kv = self._bufs.get(f"cond_kv{i}", (Bu * Lk, 2 * t.C * s), torch.bfloat16)
            run_linear(t.kv2, eb, out_bf16=kv)
            kvs.append(kv)
        bias = None
        if encoder_attention_mask is not None:
            m = encoder_attention_mask.to(self.device, non_blocking=True)
            bias = self._bufs.get("cond_bias", (Bu, Lk), torch.float32)
            if m.dtype is torch.bool:
                bias.copy_((1 - m.to(torch.float32)) * -10000.0)
            else:
                bias.copy_(m.to(torch.float32))
        extra = []
        for n, (feat, fmask) in enumerate(extra_streams):
            f = feat.to(self.device, torch.float32, non_blocking=True).contiguous()
            if f.shape[0] != Bu or f.shape[2] != D:
                raise L.TangoB200Error("extra conditioning streams must share the batch and feature width of the text states")
            Ln = f.shape[1]
            fb = self._bufs.get(f"cond_x{n}", (Bu * Ln, D * s), torch.bfloat16)
            L.cast_act(f.view(Bu * Ln, D), 1, 1, Bu * Ln, fb, split_off=D if self.split else 0)
            xk = []
            for i, t in enumerate(self.P["transformers"]):
                kvn = self._bufs.get(f"cond_x{n}kv{i}", (Bu * Ln, 2 * t.C * s), torch.bfloat16)
                run_linear(t.extra[n].kv2, fb, out_bf16=kvn)
                xk.append(kvn)
            xb = None
            if fmask is not None:
                m = fmask.to(self.device, non_blocking=True)
                xb = self._bufs.get(f"cond_x{n}bias", (Bu, Ln), torch.float32)
                xb.copy_((1 - m.to(torch.float32)) * -10000.0 if m.dtype is torch.bool else m.to(torch.float32))
            extra.append(SimpleNamespace(kvs=xk, bias=xb, Lk=Ln))
        self._cond = SimpleNamespace(kvs=kvs, bias=bias, Bu=Bu, Lk=Lk, extra=extra)

    def _arena(self, NB: int) -> StatsArena:
        a = self._arenas.get(NB)
        if a is None:
            # 1.5x: under the CFG shared prefix a few tensors exist at half batch AND full batch
            a = StatsArena(self.device, NB, self.P["stat_channels"], headroom=1.5)
            self._arenas[NB] = a
        return a

    def _transformer(self, name, t, x, st_x, NB, H, W, kv, bias, Lk, ar: StatsArena, shared_half: bool = False):
        """Transformer2DModel (transformer_2d.py:214-321) on rows; returns (out, statistics of out).
        shared_half: `x` holds only the first NB/2 images and stands for both CFG halves (identical latents and
        timestep): everything up to the self-attention output is computed once and duplicated before the
        cross-attention, the first place where the two halves see different data."""
        HW, s, sp, Cc = H * W, self.s, self.split, t.C
        so = Cc if sp else 0
        NBp = NB // 2 if shared_half else NB   # batch of the (possibly shared) prefix
        Rp, R = NBp * HW, NB * HW
        scale = 64 ** -0.5
        a = self._bufs.get("a", (Rp, Cc * s), torch.bfloat16)
        L.groupnorm(x, st_x, None, None, NBp, HW, 32, t.nw, t.nb, 1e-6, L.ACT_NONE, a, split_off=so)
        hs = self._bufs.get("hs", (R, Cc), torch.float32)
        hsp = hs[:Rp]
        run_linear(t.proj_in, a, out_f32=hsp)
        n = self._bufs.get("ln", (R, Cc * s), torch.bfloat16)
        L.layernorm(hsp, t.ln1w, t.ln1b, 1e-5, n[:Rp], split_off=so)
        qkv = self._bufs.get("qkv", (R, 3 * Cc * s), torch.bfloat16)
        run_linear(t.qkv, n[:Rp], out_bf16=qkv[:Rp])
        ao = self._bufs.get("ao", (R, Cc * s), torch.bfloat16)
        L.attention(qkv[:Rp], qkv[:Rp], qkv[:Rp], ao[:Rp], batch=NBp, heads=t.heads, Lq=HW, Lk=HW, scale=scale, q_col0=0,
                    k_col0=Cc, v_col0=2 * Cc, nsplit=s, q_lo_off=3 * Cc, k_lo_off=3 * Cc, v_lo_off=3 * Cc, split_off=so)
        run_linear(t.out1, ao[:Rp], res=hsp, out_f32=hsp)
        if shared_half:
            hs[Rp:].copy_(hsp)          # second CFG half = first half up to here
            xf = self._bufs.get(name + "_xdup", (R, Cc), torch.float32)
            xf[:Rp].copy_(x)
            xf[Rp:].copy_(x)
            x = xf
        L.layernorm(hs, t.ln2w, t.ln2b, 1e-5, n, split_off=so)
        q = self._bufs.get("q2", (R, Cc * s), torch.bfloat16)
        run_linear(t.q2, n, out_bf16=q)
        L.attention(q, kv, kv, ao, batch=NB, heads=t.heads, Lq=HW, Lk=Lk, scale=scale, q_col0=0, k_col0=0, v_col0=Cc,
                    kbias=bias, nsplit=s, q_lo_off=Cc, k_lo_off=2 * Cc, v_lo_off=2 * Cc, split_off=so)
        run_linear(t.out2, ao, res=hs, out_f32=hs)
        L.layernorm(hs, t.ln3w, t.ln3b, 1e-5, n, split_off=so)
        ff = self._bufs.get("ff", (R, 4 * Cc * s), torch.bfloat16)
        run_linear(t.ff1, n, out_bf16=ff)
        hsb = self._bufs.get("hsb", (R, Cc * s), torch.bfloat16)
        run_linear(t.ff2, ff, res=hs, out_bf16=hsb)
        out = self._bufs.get(name, (R, Cc), torch.float32)
        st_out = ar.slot(name, NB, Cc)
        run_linear(t.proj_out, hsb, res=x, out_f32=out, gn_stats=st_out, stats_hw=HW)
        return out, st_out

    def forward_rows(self, x_in: torch.Tensor, NB: int, H: int, W: int, temb: torch.Tensor, temb_ld: int,
                     out: Optional[torch.Tensor] = None, cfg_shared: bool = False) -> torch.Tensor:
        """The UNet on channels-last rows. x_in: bf16 [NB*H*W, in_ch * s] (hi | lo in split mode);
        temb: fp32 [NB, >= temb_total] rows of time_embedding_table (row stride temb_ld). Returns fp32 [NB*H*W, out_ch].
        set_conditioning() must have been called for this batch.
        cfg_shared: the two halves of the batch carry identical latents and timesteps (classifier-free guidance,
        models.py:235): conv_in, the first resnet and the first transformer up to its self-attention output — everything
        before the first cross-attention — are then computed for one half only and duplicated."""
        self._pack()
        P, cfg, sp = self.P, self.config, self.split
        c = self._cond
        if c is None or c.Bu != NB:
            raise L.TangoB200Error("set_conditioning() must be called with the same batch before forward_rows()")
        nlev = len(cfg["block_out_channels"])
        if H % (1 << (nlev - 1)) or W % (1 << (nlev - 1)):
            raise L.TangoB200Error(f"latent size {H}x{W} must be divisible by {1 << (nlev - 1)}")
        R = NB * H * W
        shared = bool(cfg_shared) and NB % 2 == 0 and bool(P["down"][0].attns)
        NBp = NB // 2 if shared else NB
        ar = self._arena(NB)
        ar.zero()                       # one fill for the GroupNorm statistics of the whole forward
        bufs = self._bufs

        def resnet(name, r, x, st_x, nb, skip=None, st_skip=None):
            return blocks.resnet(bufs, ar, sp, name, r, x, st_x, nb, ch, cw, skip, st_skip, temb[:, r.temb_off:], temb_ld)

        h, st = blocks.conv_in(bufs, ar, "conv_in", P["conv_in"], x_in, NB, H, W, NBp)
        if shared:
            h[NBp * H * W:].copy_(h[:NBp * H * W])   # the conv_in output is also a skip connection (full batch)
            st[NBp:].copy_(st[:NBp])
        skips = [(h, st)]
        ti = 0
        ch, cw = H, W

        def extras(name, t, hh, sth, idx):
            # Mustango: beat / chord transformers right after the text one (none for Tango)
            for n, tx in enumerate(t.extra):
                e = c.extra[n]
                hh, sth = self._transformer(f"{name}x{n}", tx, hh, sth, NB, ch, cw, e.kvs[idx], e.bias, e.Lk, ar)
            return hh, sth

        for i, blk in enumerate(P["down"]):
            for j, r in enumerate(blk.resnets):
                first = shared and i == 0 and j == 0
                if first:
                    hp, stp = resnet("d0r0", r, h[:NBp * H * W], st[:NBp], NBp)
                    h, st = self._transformer("d0t0", blk.attns[0], hp, stp, NB, ch, cw, c.kvs[ti], c.bias, c.Lk, ar,
                                              shared_half=True)
                    h, st = extras("d0t0", blk.attns[0], h, st, ti)
                    ti += 1
                    skips.append((h, st))
                    continue
                h, st = resnet(f"d{i}r{j}", r, h, st, NB)
                if blk.attns:
                    h, st = self._transformer(f"d{i}t{j}", blk.attns[j], h, st, NB, ch, cw, c.kvs[ti], c.bias, c.Lk, ar)
                    h, st = extras(f"d{i}t{j}", blk.attns[j], h, st, ti)
                    ti += 1
                skips.append((h, st))
            if blk.down is not None:
                h, st = blocks.downsample(bufs, ar, sp, f"d{i}ds", blk.down, h, NB, ch, cw)
                ch, cw = ch // 2, cw // 2
                skips.append((h, st))
        m = P["mid"]
        h, st = resnet("m0", m.r0, h, st, NB)
        h, st = self._transformer("mt", m.attn, h, st, NB, ch, cw, c.kvs[ti], c.bias, c.Lk, ar)
        h, st = extras("mt", m.attn, h, st, ti)
        ti += 1
        h, st = resnet("m1", m.r1, h, st, NB)
        for i, blk in enumerate(P["up"]):
            for j, r in enumerate(blk.resnets):
                skip, st_skip = skips.pop()
                h, st = resnet(f"u{i}r{j}", r, h, st, NB, skip, st_skip)
                if blk.attns:
                    h, st = self._transformer(f"u{i}t{j}", blk.attns[j], h, st, NB, ch, cw, c.kvs[ti], c.bias, c.Lk, ar)
                    h, st = extras(f"u{i}t{j}", blk.attns[j], h, st, ti)
                    ti += 1
            if blk.up is not None:
                h, st = blocks.upsample(bufs, ar, sp, f"u{i}us", blk.up, h, NB, ch, cw)
                ch, cw = 2 * ch, 2 * cw
        if out is None:
            out = bufs.get("unet_out", (R, P["conv_out"].cout), torch.float32)
        return blocks.norm_out(bufs, sp, h, st, NB, H, W, *P["norm_out"], cfg.get("norm_eps", 1e-5), P["conv_out"], out)

    # ----------------------------------------------------------------------------------------- reference-style call
    def input_rows(self, sample: torch.Tensor) -> torch.Tensor:
        """NCHW fp32 -> channels-last bf16 operand rows (hi | lo in split mode)."""
        B, Cc, H, W = sample.shape
        rows = sample.to(self.device, torch.float32).permute(0, 2, 3, 1).reshape(B * H * W, Cc).contiguous()
        xb = torch.empty(B * H * W, Cc * self.s, device=self.device, dtype=torch.bfloat16)
        L.cast_act(rows, B, H, W, xb, split_off=Cc if self.split else 0)
        return xb

    def forward(self, sample: torch.Tensor, timestep, encoder_hidden_states: torch.Tensor, class_labels=None,
                timestep_cond=None, attention_mask=None, cross_attention_kwargs=None,
                down_block_additional_residuals=None, mid_block_additional_residual=None,
                encoder_attention_mask: Optional[torch.Tensor] = None, return_dict: bool = True,
                beat_features: Optional[torch.Tensor] = None, chord_features: Optional[torch.Tensor] = None,
                beat_attention_mask: Optional[torch.Tensor] = None, chord_attention_mask: Optional[torch.Tensor] = None):
        """diffusers-compatible call: NCHW fp32 in, NCHW fp32 `.sample` out (unet_2d_condition.py:520-533). The
        beat / chord arguments are those of the Mustango variant (unet_2d_condition_music.py:536-552) and are required
        exactly when the config uses the *Music block types."""
        if attention_mask is not None or class_labels is not None or down_block_additional_residuals is not None:
            raise NotImplementedError("attention_mask / class_labels / controlnet residuals are not on the Tango path")
        self._pack()
        B, Cc, H, W = sample.shape
        ts = timestep
        if not torch.is_tensor(ts):
            ts = torch.tensor([ts], dtype=torch.float32)
        ts = ts.reshape(-1).to(torch.float32)
        ts = ts.expand(B) if ts.numel() == 1 else ts
        temb = self.time_embedding_table(ts)
        streams = ()
        if beat_features is not None or chord_features is not None:
            if beat_features is None or chord_features is None:
                raise ValueError("beat_features and chord_features must be given together")
            streams = ((beat_features, beat_attention_mask), (chord_features, chord_attention_mask))
        self.set_conditioning(encoder_hidden_states, encoder_attention_mask, extra_streams=streams)
        out = self.forward_rows(self.input_rows(sample), B, H, W, temb, temb.shape[1])
        y = out.view(B, H, W, -1).permute(0, 3, 1, 2).contiguous()
        if not return_dict:
            return (y,)
        return UNetOutput(sample=y)

    __call__ = forward
