"""Host-side pieces shared by the models: scratch buffers, the GroupNorm statistics arena, weight packing and forward of
the blocks the UNet and the VAE are built from, and the cache of captured CUDA graphs. Activations are channels-last
rows (ops.py); `split` selects the hi/lo operands of the parity mode."""
from __future__ import annotations

from collections import OrderedDict
from types import SimpleNamespace
from typing import Dict, Tuple

import torch

from . import lib as L
from .ops import PackedConv, run_conv


class Buffers:
    """Named, shape-keyed scratch tensors (allocated once, reused by every forward — CUDA-graph friendly)."""

    def __init__(self, device):
        self.device = device
        self.t: Dict[Tuple, torch.Tensor] = {}

    def get(self, name: str, shape, dtype) -> torch.Tensor:
        key = (name, tuple(shape), dtype)
        buf = self.t.get(key)
        if buf is None:
            buf = torch.zeros(shape, device=self.device, dtype=dtype)
            self.t[key] = buf
        return buf


class StatsArena:
    """fp64 per-(image, channel) GroupNorm accumulators for every norm input of one forward, carved out of ONE buffer
    so that a single fill zeroes them all at the start of the forward (slots keep their addresses: CUDA-graph safe).
    A slot [NB, C, 2] belongs to one tensor; the GEMM that produces the tensor adds its column sums from the epilogue
    (tng_conv_gemm gn_stats), the norm that consumes it — possibly twice: next layer and, as a skip connection, the up
    path — reads them. Sized for `channels` (stat_channels) at batch NB, times `headroom`."""

    def __init__(self, device, NB: int, channels: int, headroom: float = 1.0):
        self.buf = torch.zeros(int(headroom * 2 * NB * channels) + 4096, device=device, dtype=torch.float64)
        self.slots: Dict[Tuple, Tuple[int, int]] = {}
        self.used = 0

    def slot(self, name: str, NB: int, C_: int) -> torch.Tensor:
        key = (name, NB, C_)
        hit = self.slots.get(key)
        if hit is None:
            n = NB * C_ * 2
            if self.used + n > self.buf.numel():
                raise L.TangoB200Error("GroupNorm statistics arena exhausted (internal sizing error)")
            hit = (self.used, n)
            self.slots[key] = hit
            self.used += n
        return self.buf[hit[0]:hit[0] + hit[1]].view(NB, C_, 2)

    def zero(self):
        self.buf[:max(self.used, 1)].zero_()


def stat_channels(conv_in, resnets, attns, samplers) -> int:
    """Channels that carry GroupNorm statistics in one forward: conv_in, both convs of every resnet, every transformer /
    attention output and every up / down sampler conv (None entries are skipped)."""
    return (conv_in.cout + sum(2 * r.cout for r in resnets) + sum(t.C for t in attns)
            + sum(s.cout for s in samplers if s is not None))


# ------------------------------------------------------------------------------------------------------ weight packing
class Packer:
    """Packs the tensors of one state_dict for one device and precision."""

    def __init__(self, sd: Dict[str, torch.Tensor], device, split: bool):
        self.sd, self.device, self.split = sd, device, split

    def f32(self, k: str) -> torch.Tensor:
        return self.sd[k].float().contiguous().to(self.device)

    def conv(self, p: str, **kw) -> PackedConv:
        return PackedConv(self.sd[p + ".weight"], self.sd.get(p + ".bias"), split=self.split, device=self.device, **kw)

    def resnet(self, p: str, shortcut: str, eps: float) -> SimpleNamespace:
        """ResnetBlock (norm1, conv1, norm2, conv2); a 1x1 `shortcut` conv, if the block has one, is fused into conv2."""
        sd = self.sd
        r = SimpleNamespace(eps=eps)
        r.n1w, r.n1b = self.f32(p + ".norm1.weight"), self.f32(p + ".norm1.bias")
        r.n2w, r.n2b = self.f32(p + ".norm2.weight"), self.f32(p + ".norm2.bias")
        r.conv1 = self.conv(p + ".conv1")
        r.conv2 = self.conv(p + ".conv2", sc_w=sd.get(f"{p}.{shortcut}.weight"), sc_b=sd.get(f"{p}.{shortcut}.bias"))
        r.cin, r.cout = r.conv1.cin, r.conv1.cout
        return r

    def attn_block(self, p: str) -> SimpleNamespace:
        """Single-head AttnBlock: norm, 1x1 q / k / v fused into one projection, proj_out."""
        sd = self.sd
        t = SimpleNamespace(nw=self.f32(p + ".norm.weight"), nb=self.f32(p + ".norm.bias"))
        Cc = sd[p + ".q.weight"].shape[0]
        wq = torch.cat([sd[p + ".q.weight"], sd[p + ".k.weight"], sd[p + ".v.weight"]], 0).reshape(3 * Cc, Cc)
        bq = torch.cat([sd[p + ".q.bias"], sd[p + ".k.bias"], sd[p + ".v.bias"]], 0)
        t.qkv = PackedConv(wq, bq, split=self.split, device=self.device)
        t.proj = PackedConv(sd[p + ".proj_out.weight"].reshape(Cc, Cc), sd[p + ".proj_out.bias"], split=self.split,
                            device=self.device)
        t.C = Cc
        return t


# ------------------------------------------------------------------------------------------------------ forward
def resnet(bufs: Buffers, ar: StatsArena, split: bool, name: str, r, x0, st0, NB: int, H: int, W: int,
           x1=None, st1=None, rowvec=None, rowvec_ld: int = 0):
    """ResnetBlock on rows: GroupNorm + SiLU -> conv1 (+ per-image `rowvec`: the time embedding) -> GroupNorm + SiLU ->
    conv2 + residual (or + the fused shortcut of the raw input). x0 and the optional skip input x1 (concatenated along
    channels) arrive with their GroupNorm statistics st0 / st1; returns (out, statistics of out)."""
    R, HW, s = NB * H * W, H * W, 2 if split else 1
    a1 = bufs.get("a", (R, r.cin * s), torch.bfloat16)
    has_sc = r.conv2.cin_sc > 0
    raw = bufs.get("raw", (R, r.cin * s), torch.bfloat16) if has_sc else None
    L.groupnorm(x0, st0, x1, st1, NB, HW, 32, r.n1w, r.n1b, r.eps, L.ACT_SILU, a1, split_off=r.cin if split else 0,
                raw=raw, raw_split_off=r.cin if split else 0)
    h1 = bufs.get("h1", (R, r.cout), torch.float32)
    st_h1 = ar.slot(name + "_h1", NB, r.cout)
    run_conv(r.conv1, a1, NB, H, W, rowvec=rowvec, rowvec_ld=rowvec_ld, out_f32=h1, gn_stats=st_h1, stats_hw=HW)
    a2 = bufs.get("a", (R, r.cout * s), torch.bfloat16)
    L.groupnorm(h1, st_h1, None, None, NB, HW, 32, r.n2w, r.n2b, r.eps, L.ACT_SILU, a2, split_off=r.cout if split else 0)
    out = bufs.get(name, (R, r.cout), torch.float32)
    st_out = ar.slot(name, NB, r.cout)
    run_conv(r.conv2, a2, NB, H, W, sc_x=raw, res=None if has_sc else x0, out_f32=out, gn_stats=st_out, stats_hw=HW)
    return out, st_out


def downsample(bufs: Buffers, ar: StatsArena, split: bool, name: str, conv: PackedConv, x, NB: int, H: int, W: int):
    """Stride-2 conv of the fp32 rows x on the (NB, H, W) grid -> (out on the (H/2, W/2) grid, its statistics)."""
    xb = bufs.get("a", (NB * H * W, conv.cin * (2 if split else 1)), torch.bfloat16)
    L.cast_act(x, NB, H, W, xb, split_off=conv.cin if split else 0)
    out = bufs.get(name, (NB * (H // 2) * (W // 2), conv.cout), torch.float32)
    st = ar.slot(name, NB, conv.cout)
    run_conv(conv, xb, NB, H, W, out_f32=out, gn_stats=st, stats_hw=(H // 2) * (W // 2))
    return out, st


def upsample(bufs: Buffers, ar: StatsArena, split: bool, name: str, conv: PackedConv, x, NB: int, H: int, W: int):
    """Nearest x2 upsample of the fp32 rows x (in the operand cast) -> conv -> (out on the (2H, 2W) grid, statistics)."""
    xb = bufs.get("a", (NB * 4 * H * W, conv.cin * (2 if split else 1)), torch.bfloat16)
    L.cast_act(x, NB, H, W, xb, upsample2x=True, split_off=conv.cin if split else 0)
    out = bufs.get(name, (NB * 4 * H * W, conv.cout), torch.float32)
    st = ar.slot(name, NB, conv.cout)
    run_conv(conv, xb, NB, 2 * H, 2 * W, out_f32=out, gn_stats=st, stats_hw=4 * H * W)
    return out, st


def conv_in(bufs: Buffers, ar: StatsArena, name: str, conv: PackedConv, xb, NB: int, H: int, W: int, NBc=None):
    """First conv: bf16 operand rows xb -> fp32 rows + GroupNorm statistics for NB images, of which only the first NBc
    (default: all) are computed here."""
    NBc = NB if NBc is None else NBc
    out = bufs.get(name, (NB * H * W, conv.cout), torch.float32)
    st = ar.slot(name, NB, conv.cout)
    run_conv(conv, xb, NBc, H, W, out_f32=out[:NBc * H * W], gn_stats=st[:NBc], stats_hw=H * W)
    return out, st


def norm_out(bufs: Buffers, split: bool, x, st, NB: int, H: int, W: int, w, b, eps: float, conv: PackedConv, out):
    """GroupNorm + SiLU of the fp32 rows x (statistics st) -> conv into the fp32 rows `out`."""
    Cc = x.shape[1]
    a = bufs.get("a", (NB * H * W, Cc * (2 if split else 1)), torch.bfloat16)
    L.groupnorm(x, st, None, None, NB, H * W, 32, w, b, eps, L.ACT_SILU, a, split_off=Cc if split else 0)
    run_conv(conv, a, NB, H, W, out_f32=out)
    return out


# ------------------------------------------------------------------------------------------------------ CUDA graphs
class GraphCache:
    """Captured CUDA graphs by key, each with the persistent buffers it reads and writes; beyond `capacity` entries the
    least recently used one is dropped."""

    def __init__(self, capacity: int):
        self.capacity = capacity
        self._entries: OrderedDict = OrderedDict()

    def __len__(self) -> int:
        return len(self._entries)

    def clear(self):
        self._entries.clear()

    def entry(self, key, make) -> SimpleNamespace:
        """The entry of `key`; on a miss `make()` returns its persistent buffers by name, and `.graph` is None."""
        st = self._entries.get(key)
        if st is not None:
            self._entries.move_to_end(key)
            return st
        while len(self._entries) >= self.capacity:
            self._entries.popitem(last=False)
        st = self._entries[key] = SimpleNamespace(graph=None, launches=0, **make())
        return st

    @staticmethod
    def capture(st: SimpleNamespace, run) -> torch.cuda.CUDAGraph:
        """Capture `run` into st.graph unless already done: one warm-up call first (allocates the scratch buffers, sets
        kernel attributes; st.launches = its kernel launches). What run() returns under capture is st.outputs."""
        if st.graph is None:
            n0 = L.launch_count()
            run()
            st.launches = L.launch_count() - n0
            torch.cuda.synchronize()
            st.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(st.graph):
                st.outputs = run()
        return st.graph
