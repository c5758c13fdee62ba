"""AudioLDM AutoencoderKL *decoder* + HiFi-GAN vocoder on the sm_90a kernels (latents -> mel -> 16 kHz waveform).

Drop-in for the part of /root/reference/audioldm/variational_autoencoder/autoencoder.py that Tango calls
(`decode_first_stage`, `decode_to_waveform`, `.device()`, `.scale_factor`; tango.py:46-48) with the same
state_dict layout (`decoder.* post_quant_conv.* vocoder.*`; encoder / quant_conv keys are accepted and ignored —
they belong to the training path, SURVEY.md §8f).

decoder:  modules.py:650-683 (conv_in, mid res-attn-res, 3 up levels x 3 ResnetBlocks, nearest x2 + conv, norm_out,
          swish, conv_out) — same GroupNorm / wgmma conv kernels as the UNet. The single-head 512-wide mid
          AttnBlock (modules.py:204-230) is one flash-attention launch for the whole batch (tng_attention_wide: S, P and
          O in registers, the scores never reach HBM); the parity mode keeps GEMM -> row softmax -> GEMM per image.
vocoder:  hifigan/models.py:149-165 — Conv1d stacks as 1-D implicit GEMMs with leaky-ReLU / residual / 3-way average
          fused in the epilogues, ConvTranspose1d as GEMM + overlap-add gather, tanh -> int16 in one HBM kernel.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional

import numpy as np
import torch

from . import blocks
from . import lib as L
from .blocks import Buffers, GraphCache, Packer, StatsArena
from .ops import PackedConv, run_conv, run_linear
from .synth import HIFIGAN_CONFIG, VAE_CONFIG, vae_decoder_param_shapes, vae_encoder_param_shapes


class DiagonalGaussianDistribution:
    """audioldm/variational_autoencoder/distributions.py:24-41 (mean | logvar channel halves, logvar clamped to
    [-30, 20]); `sample()` draws from the torch RNG exactly as the reference does."""

    def __init__(self, parameters: torch.Tensor, deterministic: bool = False):
        self.parameters = parameters
        self.mean, self.logvar = torch.chunk(parameters, 2, dim=1)
        self.logvar = torch.clamp(self.logvar, -30.0, 20.0)
        self.deterministic = deterministic
        self.std = torch.exp(0.5 * self.logvar)
        self.var = torch.exp(self.logvar)
        if deterministic:
            self.var = self.std = torch.zeros_like(self.mean)

    def sample(self, generator=None, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        """mean + std * noise; `noise` (of the mean's shape) replaces the draw."""
        if noise is None:
            noise = torch.randn(self.mean.shape, generator=generator, device=self.mean.device, dtype=self.mean.dtype) \
                if generator is not None else torch.randn(self.mean.shape).to(self.mean.device)
        return self.mean + self.std * noise

    def mode(self) -> torch.Tensor:
        return self.mean


class AutoencoderKL:
    def __init__(self, ddconfig=None, embed_dim=None, scale_factor=1, precision: str = "bf16", **_ignored):
        self.ddconfig = dict(ddconfig or VAE_CONFIG["ddconfig"])
        self.embed_dim = embed_dim if embed_dim is not None else VAE_CONFIG["embed_dim"]
        self.scale_factor = scale_factor
        assert precision in ("bf16", "split")
        self.precision, self.split, self.s = precision, precision == "split", 2 if precision == "split" else 1
        self._device = torch.device("cpu")
        self._sd: Optional[Dict[str, torch.Tensor]] = None
        self._packed = False
        self._esd: Optional[Dict[str, torch.Tensor]] = None     # encoder.* / quant_conv.* (optional)
        self._epacked = False
        self.hifigan = dict(HIFIGAN_CONFIG)

    # ------------------------------------------------------------------------------------------ reference-style API
    def device(self):
        return self._device

    def to(self, device=None, *_a, **_k):
        if device is not None and not isinstance(device, torch.dtype):
            device = torch.device(device)
            if device != self._device:
                self._device, self._packed, self._epacked = device, False, False
        return self

    def eval(self):
        return self

    def _cfg(self):
        return {"ddconfig": self.ddconfig, "embed_dim": self.embed_dim}

    def load_state_dict(self, sd, strict: bool = True):
        want = vae_decoder_param_shapes(self._cfg())
        missing = [k for k in want if k not in sd]
        if missing:
            raise RuntimeError(f"Error(s) in loading state_dict for AutoencoderKL: missing keys {missing[:5]}...")
        for k, shp in want.items():
            if tuple(sd[k].shape) != tuple(shp):
                raise RuntimeError(f"size mismatch for {k}: {tuple(sd[k].shape)} vs {tuple(shp)}")
        self._sd = {k: sd[k].detach() for k in want}
        self._packed = False
        # encoder.* / quant_conv.* (pytorch_model_vae.bin carries them) enable encode_first_stage; they are optional
        enc = vae_encoder_param_shapes(self._cfg())
        self._esd, self._epacked = None, False
        if all(k in sd for k in enc):
            for k, shp in enc.items():
                if tuple(sd[k].shape) != tuple(shp):
                    raise RuntimeError(f"size mismatch for {k}: {tuple(sd[k].shape)} vs {tuple(shp)}")
            self._esd = {k: sd[k].detach() for k in enc}
        return SimpleNamespace(missing_keys=[], unexpected_keys=[k for k in sd if k not in want and k not in enc])

    # ------------------------------------------------------------------------------------------ packing
    def _pack(self):
        if self._packed:
            return
        if self._sd is None:
            raise L.TangoB200Error("AutoencoderKL has no weights: call load_state_dict first")
        L.require_cuda_device(self._device)
        L.load()
        sd, dev, sp = self._sd, self._device, self.split
        dd = self.ddconfig
        pk = Packer(sd, dev, sp)
        f32, conv = pk.f32, pk.conv

        def res(p):
            return pk.resnet(p, "nin_shortcut", 1e-6)

        P = SimpleNamespace()
        # post_quant_conv with the 1/scale_factor of decode_first_stage folded in (autoencoder.py:116-124,60-61)
        P.pq_w = (sd["post_quant_conv.weight"].float().reshape(sd["post_quant_conv.weight"].shape[0], -1)
                  * (1.0 / self.scale_factor)).contiguous().to(dev)
        P.pq_b = f32("post_quant_conv.bias")
        P.conv_in = conv("decoder.conv_in")
        P.mid1, P.mid2 = res("decoder.mid.block_1"), res("decoder.mid.block_2")
        P.attn = pk.attn_block("decoder.mid.attn_1")
        P.up = []
        nres = len(dd["ch_mult"])
        for lvl in reversed(range(nres)):
            blk = SimpleNamespace(res=[res(f"decoder.up.{lvl}.block.{b}") for b in range(dd["num_res_blocks"] + 1)], up=None)
            if lvl != 0:
                blk.up = conv(f"decoder.up.{lvl}.upsample.conv")
            P.up.append(blk)
        P.no_w, P.no_b = f32("decoder.norm_out.weight"), f32("decoder.norm_out.bias")
        P.conv_out = conv("decoder.conv_out")

        # ---- vocoder
        h = self.hifigan
        V = SimpleNamespace()
        V.conv_pre = conv("vocoder.conv_pre")
        V.stages = []
        nk = len(h["resblock_kernel_sizes"])
        for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
            st = SimpleNamespace(u=u, k=k, pad=(k - u) // 2)
            wt = sd[f"vocoder.ups.{i}.weight"]  # (Cin, Cout, k)
            st.cin, st.cout = wt.shape[0], wt.shape[1]
            st.up = PackedConv(wt.permute(2, 1, 0).reshape(k * st.cout, st.cin), None, split=sp, device=dev)
            st.up_bias = f32(f"vocoder.ups.{i}.bias")
            st.blocks = []
            for j, rk in enumerate(h["resblock_kernel_sizes"]):
                rb = SimpleNamespace(c1=[], c2=[])
                p = f"vocoder.resblocks.{i * nk + j}"
                for di, d in enumerate(h["resblock_dilation_sizes"][j]):
                    rb.c1.append(conv(f"{p}.convs1.{di}", dilation=d))
                    rb.c2.append(conv(f"{p}.convs2.{di}"))
                st.blocks.append(rb)
            V.stages.append(st)
        V.conv_post = conv("vocoder.conv_post")
        res_all = [P.mid1, P.mid2] + [r for blk in P.up for r in blk.res]
        P.stat_channels = blocks.stat_channels(P.conv_in, res_all, [P.attn], [blk.up for blk in P.up])
        self.P, self.V = P, V
        self._bufs = Buffers(dev)
        self._arenas = {}
        self._graphs = GraphCache(4)
        self._packed = True

    def _arena(self, tag: str, NB: int, channels: int) -> StatsArena:
        """GroupNorm statistics arena of one decode / encode call (see blocks.StatsArena)."""
        key = (tag, NB)
        a = self._arenas.get(key)
        if a is None:
            a = StatsArena(self._device, NB, channels)
            self._arenas[key] = a
        a.zero()
        return a

    # ------------------------------------------------------------------------------------------ decoder
    def _attn(self, x, st, NB, H, W, ar, t=None):
        """modules.py:204-230: softmax(q k^T / sqrt(C)) v over the H*W positions of each image, one head.
        `t`: packed attention weights (default: the decoder's mid block). Returns (out, stats of out)."""
        t = self.P.attn if t is None else t
        R, HW, s, sp, Cc = NB * H * W, H * W, self.s, self.split, t.C
        if HW % 64:
            raise L.TangoB200Error("VAE attention needs H*W to be a multiple of 64")
        a = self._bufs.get("a", (R, Cc * s), torch.bfloat16)
        L.groupnorm(x, st, None, None, NB, HW, 32, t.nw, t.nb, 1e-6, L.ACT_NONE, a, split_off=Cc if sp else 0)
        qkv = self._bufs.get("vqkv", (R, 3 * Cc * s), torch.bfloat16)  # [q k v | q_lo k_lo v_lo]
        run_linear(t.qkv, a, out_bf16=qkv)
        o = self._bufs.get("vo", (R, Cc * s), torch.bfloat16)
        if not sp and Cc == 512 and HW % 128 == 0:
            # perf mode: one flash-attention launch for the whole batch, the [HW, HW] scores never leave the SM
            L.attention_wide(qkv, qkv, qkv, o, batch=NB, L=HW, dim=Cc, scale=float(Cc) ** -0.5, q_col0=0, k_col0=Cc,
                             v_col0=2 * Cc)
            out = self._bufs.get("vattn", (R, Cc), torch.float32)
            st_out = ar.slot("vattn", NB, Cc)
            run_linear(t.proj, o, res=x, out_f32=out, gn_stats=st_out, stats_hw=HW)
            return out, st_out
        # parity mode (hi/lo split operands): scores through HBM, image by image — GEMM -> row softmax -> GEMM
        S = self._bufs.get("vS", (HW, HW), torch.float32)
        Pm = self._bufs.get("vP", (HW, HW * s), torch.bfloat16)
        vt = self._bufs.get("vVt", (Cc, HW * s), torch.bfloat16)
        nkb_c, nkb_hw = Cc // 64, HW // 64
        lo = 3 * Cc
        for b in range(NB):
            rows = qkv[b * HW:(b + 1) * HW]
            av = L.View(rows, rows.shape[1], HW, 1, 1, rows.stride(0), HW * rows.stride(0), HW * rows.stride(0))
            # S = q k^T: A columns [0,C) (q), B = the same rows read as a [HW, ld] matrix, columns [C,2C) (k)
            if sp:
                g = [(0, 0, 0, 0, Cc, nkb_c), (0, lo, 0, 0, Cc, nkb_c), (0, 0, 0, 0, lo + Cc, nkb_c)]
            else:
                g = [(0, 0, 0, 0, Cc, nkb_c)]
            L.conv_gemm([av], g, rows, HW, 1, 1, out_f32=S)
            L.softmax_rows(S, float(Cc) ** -0.5, Pm, L=HW, split_off=HW if sp else 0)
            # V^T (K-major B operand of P v): hi (and lo) halves transposed separately
            L.transpose_bf16(rows[:, 2 * Cc:3 * Cc], 1, HW, Cc, vt[:, :HW])
            if sp:
                L.transpose_bf16(rows[:, lo + 2 * Cc:lo + 3 * Cc], 1, HW, Cc, vt[:, HW:])
            pv = L.View(Pm, Pm.shape[1], HW, 1, 1, Pm.stride(0), HW * Pm.stride(0), HW * Pm.stride(0))
            if sp:
                g = [(0, 0, 0, 0, 0, nkb_hw), (0, HW, 0, 0, 0, nkb_hw), (0, 0, 0, 0, HW, nkb_hw)]
            else:
                g = [(0, 0, 0, 0, 0, nkb_hw)]
            ob = o[b * HW:(b + 1) * HW]
            L.conv_gemm([pv], g, vt, HW, 1, 1, out_bf16=ob, split_off=Cc if sp else 0)
        out = self._bufs.get("vattn", (R, Cc), torch.float32)
        st_out = ar.slot("vattn", NB, Cc)
        run_linear(t.proj, o, res=x, out_f32=out, gn_stats=st_out, stats_hw=HW)
        return out, st_out

    def decode_rows(self, z_rows: torch.Tensor, NB: int, H: int, W: int) -> torch.Tensor:
        """z_rows fp32 [NB*H*W, 8] (channels-last latents) -> mel fp32 [NB*4H*4W, 1] (== [NB*4H, 64] for W = 16)."""
        self._pack()
        P, s, sp = self.P, self.s, self.split
        R = NB * H * W
        zc = P.pq_w.shape[0]
        z1 = self._bufs.get("vz", (R, zc), torch.float32)
        L.linear_f32(z_rows, P.pq_w, P.pq_b, z1)
        zb = self._bufs.get("vzb", (R, zc * s), torch.bfloat16)
        L.cast_act(z1, NB, H, W, zb, split_off=zc if sp else 0)
        ar = self._arena("dec", NB, P.stat_channels)
        bufs = self._bufs
        h, st = blocks.conv_in(bufs, ar, "vconv_in", P.conv_in, zb, NB, H, W)
        h, st = blocks.resnet(bufs, ar, sp, "vmid1", P.mid1, h, st, NB, H, W)
        h, st = self._attn(h, st, NB, H, W, ar)
        h, st = blocks.resnet(bufs, ar, sp, "vmid2", P.mid2, h, st, NB, H, W)
        ch, cw = H, W
        for li, blk in enumerate(P.up):
            for bi, r in enumerate(blk.res):
                h, st = blocks.resnet(bufs, ar, sp, f"vup{li}_{bi}", r, h, st, NB, ch, cw)
            if blk.up is not None:
                h, st = blocks.upsample(bufs, ar, sp, f"vups{li}", blk.up, h, NB, ch, cw)
                ch, cw = 2 * ch, 2 * cw
        mel = bufs.get("vmel", (NB * ch * cw, P.conv_out.cout), torch.float32)
        return blocks.norm_out(bufs, sp, h, st, NB, ch, cw, P.no_w, P.no_b, 1e-6, P.conv_out, mel)

    def decode_rows_to_waveform(self, z_rows: torch.Tensor, NB: int, H: int, W: int, use_cuda_graph: bool = True):
        """decode_first_stage + decode_to_waveform on rows: fp32 [NB*H*W, 8] latents -> (wave fp32 [NB, L], int16
        [NB, L]) on the device. The ~600 launches of the decoder and the vocoder are captured once per shape into a CUDA
        graph (all operands live in persistent buffers) and replayed afterwards."""
        self._pack()

        def run(z):
            mel = self.decode_rows(z, NB, H, W)
            return self.vocoder_rows(mel.view(NB * 4 * H, 4 * W), NB, 4 * H)

        if not use_cuda_graph:
            return run(z_rows)
        st = self._graphs.entry((NB, H, W),
                                lambda: dict(zin=self._bufs.get("graph_zin", tuple(z_rows.shape), torch.float32)))
        st.zin.copy_(z_rows)
        self._graphs.capture(st, lambda: run(st.zin)).replay()
        return st.outputs

    def decode_first_stage(self, z: torch.Tensor, predict_cids=False, force_not_quantize=False) -> torch.Tensor:
        """(B, 8, T/4, 16) latents -> (B, 1, T, 64) log-mel (autoencoder.py:116-124)."""
        if predict_cids:
            raise NotImplementedError("predict_cids is not on the Tango path")
        L.require_cuda(z)   # no CPU fallback
        B, Cc, H, W = z.shape
        rows = z.float().permute(0, 2, 3, 1).reshape(B * H * W, Cc).contiguous()
        mel = self.decode_rows(rows, B, H, W)
        oc = mel.shape[1]
        return mel.view(B, 4 * H, 4 * W, oc).permute(0, 3, 1, 2).contiguous()

    # ------------------------------------------------------------------------------------------ encoder
    # SURVEY.md section 8(f).2 — the step in front of the diffusion model for training / audio-to-audio:
    # audioldm/variational_autoencoder/modules.py:419-543 (Encoder), :76-94 (Downsample), autoencoder.py:52-58,110-112
    # (encode / encode_first_stage), distributions.py:24-41. Same building blocks as the decoder; the stride-2
    # Downsample pads one row / column at the END of each axis, which is PackedConv(stride=2, pad=0) on the TMA zero fill.
    def _pack_encoder(self):
        if self._epacked:
            return
        self._pack()
        if self._esd is None:
            raise L.TangoB200Error("AutoencoderKL was loaded without encoder.* / quant_conv.* weights")
        sd, dev, sp, dd = self._esd, self._device, self.split, self.ddconfig
        pk = Packer(sd, dev, sp)
        f32, conv = pk.f32, pk.conv

        def res(p):
            return pk.resnet(p, "nin_shortcut", 1e-6)

        E = SimpleNamespace()
        w_in = sd["encoder.conv_in.weight"].float()
        E.cin_pad = 8                                   # activation views need a multiple of 8 channels: zero-pad 1 -> 8
        E.conv_in = PackedConv(torch.nn.functional.pad(w_in, (0, 0, 0, 0, 0, E.cin_pad - w_in.shape[1])),
                               sd["encoder.conv_in.bias"], split=sp, device=dev)
        E.down = []
        nres = len(dd["ch_mult"])
        for lvl in range(nres):
            blk = SimpleNamespace(res=[res(f"encoder.down.{lvl}.block.{b}") for b in range(dd["num_res_blocks"])], down=None)
            if lvl != nres - 1:
                blk.down = conv(f"encoder.down.{lvl}.downsample.conv", stride=2, pad=0)
            E.down.append(blk)
        E.mid1, E.mid2 = res("encoder.mid.block_1"), res("encoder.mid.block_2")
        E.attn = pk.attn_block("encoder.mid.attn_1")
        E.no_w, E.no_b = f32("encoder.norm_out.weight"), f32("encoder.norm_out.bias")
        E.conv_out = conv("encoder.conv_out")
        E.q_w = sd["quant_conv.weight"].float().reshape(sd["quant_conv.weight"].shape[0], -1).contiguous().to(dev)
        E.q_b = f32("quant_conv.bias")
        eres = [r for blk in E.down for r in blk.res] + [E.mid1, E.mid2]
        E.stat_channels = blocks.stat_channels(E.conv_in, eres, [E.attn], [blk.down for blk in E.down])
        self.E = E
        self._epacked = True

    def encode_rows(self, mel_rows: torch.Tensor, NB: int, H: int, W: int) -> torch.Tensor:
        """mel_rows fp32 [NB*H*W, 1] (channels-last log-mel, H = frames, W = 64 bins) -> moments fp32
        [NB*(H/4)*(W/4), 2*embed_dim] (mean | logvar channels of the posterior)."""
        self._pack_encoder()
        E, s, sp = self.E, self.s, self.split
        R = NB * H * W
        x8 = torch.zeros(R, E.cin_pad, device=mel_rows.device, dtype=torch.float32)
        x8[:, :mel_rows.shape[1]] = mel_rows
        xb = self._bufs.get("a", (R, E.cin_pad * s), torch.bfloat16)
        L.cast_act(x8, NB, H, W, xb, split_off=E.cin_pad if sp else 0)
        ar = self._arena("enc", NB, E.stat_channels)
        bufs = self._bufs
        h, st = blocks.conv_in(bufs, ar, "econv_in", E.conv_in, xb, NB, H, W)
        ch, cw = H, W
        for li, blk in enumerate(E.down):
            for bi, r in enumerate(blk.res):
                h, st = blocks.resnet(bufs, ar, sp, f"edown{li}_{bi}", r, h, st, NB, ch, cw)
            if blk.down is not None:
                h, st = blocks.downsample(bufs, ar, sp, f"edown{li}_ds", blk.down, h, NB, ch, cw)
                ch, cw = ch // 2, cw // 2
        h, st = blocks.resnet(bufs, ar, sp, "emid1", E.mid1, h, st, NB, ch, cw)
        h, st = self._attn(h, st, NB, ch, cw, ar, E.attn)
        h, st = blocks.resnet(bufs, ar, sp, "emid2", E.mid2, h, st, NB, ch, cw)
        mom = bufs.get("emom", (NB * ch * cw, E.conv_out.cout), torch.float32)
        blocks.norm_out(bufs, sp, h, st, NB, ch, cw, E.no_w, E.no_b, 1e-6, E.conv_out, mom)
        out = self._bufs.get("emoments", (NB * ch * cw, E.q_w.shape[0]), torch.float32)
        L.linear_f32(mom, E.q_w, E.q_b, out)
        return out

    def encode(self, x: torch.Tensor) -> "DiagonalGaussianDistribution":
        """(B, 1, T, 64) log-mel -> posterior over (B, embed_dim, T/4, 16) latents (autoencoder.py:52-58)."""
        L.require_cuda(x)   # no CPU fallback
        B, Cc, T, Fq = x.shape
        if Cc != 1 or T % 16 or Fq % 4:
            raise L.TangoB200Error("encode expects (B, 1, T, F) with T a multiple of 16 and F of 4")
        rows = x.float().permute(0, 2, 3, 1).reshape(B * T * Fq, 1).contiguous()
        mom = self.encode_rows(rows, B, T, Fq)
        return DiagonalGaussianDistribution(mom.view(B, T // 4, Fq // 4, -1).permute(0, 3, 1, 2).contiguous())

    def encode_first_stage(self, x: torch.Tensor) -> "DiagonalGaussianDistribution":
        return self.encode(x)

    @property
    def has_encoder(self) -> bool:
        return self._esd is not None

    def get_first_stage_encoding(self, encoder_posterior) -> torch.Tensor:
        """autoencoder.py:126-135: scale_factor * (a sample of the posterior, or the given latents) — the latent space
        the diffusion UNet was trained in."""
        if isinstance(encoder_posterior, DiagonalGaussianDistribution):
            z = encoder_posterior.sample()
        elif isinstance(encoder_posterior, torch.Tensor):
            z = encoder_posterior
        else:
            raise NotImplementedError(f"encoder_posterior of type '{type(encoder_posterior)}' not yet implemented")
        return self.scale_factor * z

    # ------------------------------------------------------------------------------------------ vocoder
    def vocoder_rows(self, mel_rows: torch.Tensor, B: int, T: int):
        """mel_rows fp32 [B*T, 64] -> (wave fp32 [B, L], int16 [B, L]) on the device."""
        self._pack()
        V, s, sp = self.V, self.s, self.split
        nm = mel_rows.shape[1]
        xb = self._bufs.get("hb", (B * T, nm * s), torch.bfloat16)
        L.cast_act(mel_rows, B, 1, T, xb, split_off=nm if sp else 0)
        x = self._bufs.get("hx_pre", (B * T, V.conv_pre.cout), torch.float32)
        run_conv(V.conv_pre, xb, B, 1, T, out_f32=x)
        Lc = T
        for si, st in enumerate(V.stages):
            xb = self._bufs.get("hb", (B * Lc, st.cin * s), torch.bfloat16)
            L.cast_act(x, B, 1, Lc, xb, act=L.ACT_LRELU, act_param=0.1, split_off=st.cin if sp else 0)
            Y = self._bufs.get("hY", (B * Lc, st.k * st.cout), torch.float32)
            run_conv(st.up, xb, B, 1, Lc, out_f32=Y)
            Lo = (Lc - 1) * st.u - 2 * st.pad + st.k
            x = self._bufs.get(f"hx{si}", (B * Lo, st.cout), torch.float32)
            L.convt_gather(Y, B, Lc, st.k, st.cout, st.u, st.pad, Lo, st.up_bias, x)
            Lc = Lo
            xs = self._bufs.get(f"hxs{si}", (B * Lc, st.cout), torch.float32)
            C_ = st.cout
            so = C_ if sp else 0
            x_act = self._bufs.get("hxa", (B * Lc, C_ * s), torch.bfloat16)  # lrelu(x): shared first operand of the 3 blocks
            L.cast_act(x, B, 1, Lc, x_act, act=L.ACT_LRELU, act_param=0.1, split_off=so)
            nb = len(st.blocks)
            for j, rb in enumerate(st.blocks):
                cur, cur_act = x, x_act
                rbuf = self._bufs.get("hrb", (B * Lc, C_), torch.float32)
                ract = self._bufs.get("hra", (B * Lc, C_ * s), torch.bfloat16)
                xt = self._bufs.get("hxt", (B * Lc, C_ * s), torch.bfloat16)
                nd = len(rb.c1)
                for di in range(nd):
                    # xt = lrelu(conv1(lrelu(cur)))  (models.py:98-100), kept only as the bf16 operand of conv2
                    run_conv(rb.c1[di], cur_act, B, 1, Lc, out_bf16=xt, act=L.ACT_LRELU, act_param=0.1)
                    if di < nd - 1:
                        # cur = conv2(xt) + cur ; next operand lrelu(cur) comes from the same epilogue
                        run_conv(rb.c2[di], xt, B, 1, Lc, res=cur, out_f32=rbuf, out_bf16=ract, act=L.ACT_LRELU,
                                 act_param=0.1)
                        cur, cur_act = rbuf, ract
                    else:
                        # last conv of the block: xs (+)= (conv2(xt) + cur) / num_kernels  (models.py:154-160)
                        run_conv(rb.c2[di], xt, B, 1, Lc, res=cur, alpha=1.0 / nb, accumulate=j > 0, out_f32=xs)
            x = xs
        cin = V.conv_post.cin
        xb = self._bufs.get("hb", (B * Lc, cin * s), torch.bfloat16)
        L.cast_act(x, B, 1, Lc, xb, act=L.ACT_LRELU, act_param=0.01, split_off=cin if sp else 0)  # F.leaky_relu default
        y = self._bufs.get("hpost", (B * Lc, 1), torch.float32)
        run_conv(V.conv_post, xb, B, 1, Lc, out_f32=y)
        wf = self._bufs.get("hwave_f", (B, Lc), torch.float32)
        wi = self._bufs.get("hwave_i", (B, Lc), torch.int16)
        L.tanh_to_i16(y, B * Lc, 1, wf, wi)
        return wf, wi

    def decode_to_waveform(self, dec: torch.Tensor) -> np.ndarray:
        """(B, 1, T, 64) mel -> int16 numpy (B, L) (autoencoder.py:66-69; hifigan/utilities.py:76-86)."""
        L.require_cuda(dec)   # no CPU fallback
        B, _, T, nm = dec.shape
        rows = dec.float().reshape(B * T, nm).contiguous()  # squeeze(1).permute(0,2,1) in channels-last = same memory
        _, wi = self.vocoder_rows(rows, B, T)
        return wi.cpu().numpy()
