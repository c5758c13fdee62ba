"""FLAN-T5 encoder on the tango_b200 kernels — the text-conditioning front-end of the hot path (SURVEY.md section 8(f).1).

Mirrors `transformers.T5EncoderModel` as the reference uses it: built at /root/reference/models.py:98-100, called as
`self.text_encoder(input_ids=..., attention_mask=...)[0]` in models.py:129-147 (encode_text) and :266-305
(encode_text_classifier_free). State_dict keys and config fields are those of T5EncoderModel (`shared.weight`,
`encoder.block.{i}.layer.0.SelfAttention.{q,k,v,o}.weight`, `...relative_attention_bias.weight`,
`encoder.block.{i}.layer.{0,1}.layer_norm.weight`, `...DenseReluDense.{wi_0,wi_1,wo}.weight`,
`encoder.final_layer_norm.weight`), so `text_encoder.*` of pytorch_model_main.bin loads unchanged.

Per block: tng_rmsnorm -> fused q|k|v projection (tng_conv_gemm, fp32 out) -> tng_rel_attention (relative position
bias + key mask, no score scaling) -> o projection with the residual add in the GEMM epilogue -> tng_rmsnorm ->
wi_1|wi_0 projection with the gated tanh-GELU fused in the epilogue -> wo projection + residual.
The residual stream stays fp32; GEMM operands are bf16 (perf mode) or hi+lo bf16 pairs (precision="split").
"""
from __future__ import annotations

import json
import math
import os
from types import SimpleNamespace
from typing import Dict, Optional

import torch

from . import lib as L
from .blocks import GraphCache
from .ops import PackedConv, run_linear


class T5Output(tuple):
    """`model(...)[0]` and `.last_hidden_state`, like transformers' BaseModelOutput."""

    def __new__(cls, last_hidden_state):
        return super().__new__(cls, (last_hidden_state,))

    @property
    def last_hidden_state(self):
        return self[0]


def relative_position_buckets(L_: int, num_buckets: int, max_distance: int) -> torch.Tensor:
    """bucket[key - query + L - 1] for the bidirectional encoder attention (modeling_t5.py
    T5Attention._relative_position_bucket): half of the buckets per sign; within a sign the first half are exact
    offsets, the rest logarithmic bins up to max_distance. Host-side table (2L-1 integers), built once per length."""
    rel = torch.arange(-(L_ - 1), L_, dtype=torch.long)
    half = num_buckets // 2
    exact = half // 2
    n = rel.abs()
    log_bin = exact + (torch.log(n.float() / exact) / math.log(max_distance / exact) * (half - exact)).to(torch.long)
    log_bin = torch.clamp(log_bin, max=half - 1)
    return (rel > 0).to(torch.long) * half + torch.where(n < exact, n, log_bin)


class T5EncoderModel:
    config_keys = ("vocab_size", "d_model", "d_kv", "num_heads", "d_ff", "num_layers",
                   "relative_attention_num_buckets", "relative_attention_max_distance", "layer_norm_epsilon",
                   "feed_forward_proj")

    def __init__(self, config: dict, precision: str = "bf16"):
        cfg = dict(config)
        cfg.setdefault("relative_attention_num_buckets", 32)
        cfg.setdefault("relative_attention_max_distance", 128)
        cfg.setdefault("layer_norm_epsilon", 1e-6)
        cfg.setdefault("feed_forward_proj", "gated-gelu")
        if cfg["feed_forward_proj"] != "gated-gelu":
            raise NotImplementedError("only the FLAN-T5 (gated-gelu) feed-forward is on the Tango path")
        if cfg["d_kv"] != 64:
            raise NotImplementedError("attention head width must be 64 (FLAN-T5 large / xl)")
        if cfg["d_model"] % 64 or cfg["d_ff"] % 128 or cfg["d_model"] > 2048:
            raise NotImplementedError("d_model must be a multiple of 64 (<= 2048) and d_ff a multiple of 128")
        assert precision in ("bf16", "split")
        self.config = SimpleNamespace(**cfg)
        self.cfg = cfg
        self.precision, self.split = precision, precision == "split"
        self.device = torch.device("cpu")
        self.dtype = torch.float32
        self._sd: Optional[Dict[str, torch.Tensor]] = None
        self._packed = False
        self._relbias = {}
        self._graphs = GraphCache(8)
        self.use_cuda_graph = True      # one graph per (batch, padded length); off under the CPU orchestration tests

    # ----------------------------------------------------------------------------------------- transformers-style API
    @classmethod
    def from_config(cls, config: dict, precision: str = "bf16") -> "T5EncoderModel":
        return cls(config, precision=precision)

    @classmethod
    def from_pretrained(cls, path: str, precision: str = "bf16", **_kw) -> "T5EncoderModel":
        """Local snapshot directory only (config.json + pytorch_model.bin | model.safetensors); no hub access."""
        with open(os.path.join(path, "config.json")) as f:
            cfg = json.load(f)
        m = cls({k: cfg[k] for k in cls.config_keys if k in cfg}, precision=precision)
        st = os.path.join(path, "model.safetensors")
        if os.path.exists(st):
            from safetensors.torch import load_file
            sd = load_file(st)
        else:
            sd = torch.load(os.path.join(path, "pytorch_model.bin"), map_location="cpu")
        m.load_state_dict(sd, strict=False)
        return m

    def parameters_shapes(self):
        from .synth import t5_encoder_param_shapes
        return t5_encoder_param_shapes(self.cfg)

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        sd = dict(sd)
        if "shared.weight" not in sd and "encoder.embed_tokens.weight" in sd:
            sd["shared.weight"] = sd["encoder.embed_tokens.weight"]
        want = self.parameters_shapes()
        ignorable = ("encoder.embed_tokens.weight",)          # tied copy of shared.weight
        missing = [k for k in want if k not in sd]
        unexpected = [k for k in sd if k not in want and k not in ignorable]
        if missing or (strict and unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:5]}..., unexpected {unexpected[:5]}...")
        for k, shp in want.items():
            if tuple(sd[k].shape) != tuple(shp):
                raise RuntimeError(f"size mismatch for {k}: {tuple(sd[k].shape)} vs {tuple(shp)}")
        self._sd = {k: sd[k].detach() for k in want}
        self._packed = False
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def to(self, device=None, *_a, **_k):
        if device is not None and not isinstance(device, torch.dtype):
            device = torch.device(device)
            if device != self.device:
                self.device, self._packed = device, False
        return self

    def eval(self):
        return self

    # ----------------------------------------------------------------------------------------- packing
    def _pack(self):
        if self._packed:
            return
        if self._sd is None:
            raise L.TangoB200Error("T5EncoderModel has no weights: call load_state_dict first")
        L.require_cuda_device(self.device)
        L.load()
        sd, dev, sp, cfg = self._sd, self.device, self.split, self.cfg
        f32 = lambda k: sd[k].detach().float().contiguous().to(dev)
        self.emb = f32("shared.weight")
        self.rel_table = f32("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight")  # [buckets, heads]
        self.final_ln = f32("encoder.final_layer_norm.weight")
        self.blocks = []
        for i in range(cfg["num_layers"]):
            p = f"encoder.block.{i}.layer."
            b = SimpleNamespace()
            b.ln0, b.ln1 = f32(p + "0.layer_norm.weight"), f32(p + "1.layer_norm.weight")
            wqkv = torch.cat([sd[p + f"0.SelfAttention.{n}.weight"].float() for n in ("q", "k", "v")], 0)
            b.qkv = PackedConv(wqkv, None, split=sp, device=dev)
            b.o = PackedConv(sd[p + "0.SelfAttention.o.weight"], None, split=sp, device=dev)
            # gated feed-forward: out = wi_1(x) * gelu_new(wi_0(x)) -> [hidden | gate] rows = [wi_1 | wi_0]
            wff = torch.cat([sd[p + "1.DenseReluDense.wi_1.weight"].float(), sd[p + "1.DenseReluDense.wi_0.weight"].float()], 0)
            b.ff1 = PackedConv(wff, None, split=sp, device=dev, geglu_bn=256 if cfg["d_ff"] % 128 == 0 else 128,
                               geglu_tanh=True)
            b.ff2 = PackedConv(sd[p + "1.DenseReluDense.wo.weight"], None, split=sp, device=dev)
            self.blocks.append(b)
        self._relbias = {}
        self._graphs.clear()
        self._packed = True

    def _relbias_for(self, L_: int) -> torch.Tensor:
        """fp32 [heads, 2L-1]: relative_attention_bias[bucket(key - query), head] (T5Attention.compute_bias)."""
        t = self._relbias.get(L_)
        if t is None:
            idx = relative_position_buckets(L_, self.cfg["relative_attention_num_buckets"],
                                            self.cfg["relative_attention_max_distance"]).to(self.device)
            t = self.rel_table.index_select(0, idx).t().contiguous()
            self._relbias[L_] = t
        return t

    # ----------------------------------------------------------------------------------------- forward
    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, **_kw) -> T5Output:
        self._pack()
        L.require_cuda(input_ids)
        cfg, dev, s = self.cfg, self.device, (2 if self.split else 1)
        B, Lt = input_ids.shape
        ids = input_ids.to(torch.int64).contiguous()
        lo, hi = int(ids.min()), int(ids.max())
        if lo < 0 or hi >= cfg["vocab_size"]:
            raise IndexError(f"token id out of range [0, {cfg['vocab_size']}): min {lo}, max {hi}")
        d, H, ff = cfg["d_model"], cfg["num_heads"], cfg["d_ff"]
        inner, rows, eps = H * 64, B * Lt, float(cfg["layer_norm_epsilon"])
        # persistent operands: the ~170 launches of the stack are captured once per (batch, length) into a CUDA graph
        st = self._graphs.entry((B, Lt, attention_mask is not None), lambda: dict(
            ids=torch.zeros(rows, device=dev, dtype=torch.int64),
            kbias=torch.zeros(B, Lt, device=dev, dtype=torch.float32) if attention_mask is not None else None,
            x=torch.empty(rows, d, device=dev, dtype=torch.float32),
            n=torch.empty(rows, s * d, device=dev, dtype=torch.bfloat16),
            qkv=torch.empty(rows, 3 * inner, device=dev, dtype=torch.float32),
            ctx=torch.empty(rows, s * inner, device=dev, dtype=torch.bfloat16),
            hff=torch.empty(rows, s * ff, device=dev, dtype=torch.bfloat16),
            out=torch.empty(rows, d, device=dev, dtype=torch.float32)))
        st.ids.copy_(ids.view(-1))
        if st.kbias is not None:
            # get_extended_attention_mask: (1 - mask) * finfo.min, added to the position bias
            st.kbias.copy_((1.0 - attention_mask.to(dev).float()) * torch.finfo(torch.float32).min)
        relbias = self._relbias_for(Lt)
        so_d, so_i = (d if self.split else 0), (inner if self.split else 0)

        def run():
            x, n, qkv, ctx, hff = st.x, st.n, st.qkv, st.ctx, st.hff
            L.gather_rows(self.emb, st.ids, x)
            for b in self.blocks:
                L.rmsnorm(x, b.ln0, eps, n, split_off=so_d)
                run_linear(b.qkv, n, out_f32=qkv)
                L.rel_attention(qkv, relbias, st.kbias, ctx, batch=B, heads=H, L=Lt, q_col0=0, k_col0=inner,
                                v_col0=2 * inner, split_off=so_i)
                run_linear(b.o, ctx, res=x, out_f32=x)
                L.rmsnorm(x, b.ln1, eps, n, split_off=so_d)
                run_linear(b.ff1, n, out_bf16=hff)
                run_linear(b.ff2, hff, res=x, out_f32=x)
            # final T5LayerNorm in fp32: it is the tensor handed to the UNet's cross-attention K/V projections
            L.rmsnorm(x, self.final_ln, eps, y_f32=st.out)

        if not (self.use_cuda_graph and dev.type == "cuda"):
            run()
        else:
            self._graphs.capture(st, run).replay()
        return T5Output(st.out.view(B, Lt, d).clone())

    __call__ = forward
