"""Plain-Python statement of the persistent GEMM's planner and epilogue dispatch (TEST INFRASTRUCTURE ONLY).

`plan(d, sms)` restates plan_gemm / tile_m / full_m_tiles of tango_b200/csrc/gemm_tc.cu (the N tile, the M tile, split-K,
fast_epi, where the GroupNorm statistics come from, and every TNG_EINVAL rejection); `cells(d, sms)` walks the launch's
work items as gemm_tc_kernel does (nvalid, the `full` test, the output mode) and returns the epilogue cells it runs:

    (BN, BM, body, feature)

body: FULL:<mode> (mode bits 1 residual, 2 fp32 output, 4 bf16 output), VEC, SCALAR or one of the GEGLU forms;
feature: a run-time property that changes what that body executes (the per-warp or per-slot row vector, accumulate,
the activation, the hi/lo split, the output mode of the VEC / SCALAR bodies, split-K red.add over an even or odd number
of K blocks, fused or after-pass statistics, a non-full tile reached by a CTA that ran a FULL one before), or "run".

REACHABLE is the matrix of every cell the dispatch can reach; EXCLUDED names the reason for every other cell of the
product. Descriptors are `Desc` objects: the fields of tng_gemm_desc, pointers as integer addresses (0 = NULL), so that
the statement runs without a device; `desc_of` builds one from the arguments of tango_b200.lib.conv_gemm.
"""
from __future__ import annotations

import ctypes
import struct
from dataclasses import dataclass, field

from tango_b200 import lib as L

BK = 64
BNS = (32, 64, 128, 160, 256)
BMS = (128, 256)
INSTANTIATIONS = tuple((bn, 128) for bn in BNS) + ((160, 256),)
MODES = (2, 3, 4, 5, 6, 7)
GEGLU_BODIES = ("GEGLU:erf-full", "GEGLU:erf-partial", "GEGLU:erf-hilo", "GEGLU:tanh", "GEGLU:tanh-hilo")
BODIES = tuple(f"FULL:{m}" for m in MODES) + ("VEC", "SCALAR") + GEGLU_BODIES
FEATURES = ("run", "rowvec:warp", "rowvec:slot", "accumulate", "act:silu", "act:lrelu", "hilo") + \
    tuple(f"mode:{m}" for m in MODES) + ("red:even", "red:odd", "stats:fused", "stats:after", "after-full")
GEGLU_ACTS = (L.ACT_GEGLU, L.ACT_GEGLU_TANH)


@dataclass
class Desc:
    """tng_gemm_desc with integer pointers. a: [(ptr, C, W, H, NB, s_w, s_h, s_n)]; g: [(view, a_c0, dw, dh, b_k0, nkb)]."""
    a: list
    g: list
    W: int
    H: int
    NB: int
    Ncols: int
    Ktot: int
    b: int = 0
    ldb: int = 0
    bias: int = 0
    rowvec: int = 0
    rowvec_ld: int = 0
    res: int = 0
    res_dtype: int = L.DT_F32
    ldr: int = 0
    alpha: float = 1.0
    accumulate: int = 0
    out_f32: int = 0
    ld_f32: int = 0
    out_bf16: int = 0
    ld_bf16: int = 0
    act: int = L.ACT_NONE
    act_param: float = 0.0
    split_off: int = 0
    block_n: int = 0
    gn_stats: int = 0
    stats_hw: int = 0
    n_aviews: int = field(default=-1)
    n_groups: int = field(default=-1)

    def __post_init__(self):
        if self.n_aviews < 0:
            self.n_aviews = len(self.a)
        if self.n_groups < 0:
            self.n_groups = len(self.g)

    def ctypes(self) -> L.GemmDesc:
        d = L.GemmDesc()
        for i, v in enumerate(self.a[:L.MAX_AVIEWS]):
            d.a[i] = L.AView(*v)
        for i, g in enumerate(self.g[:L.MAX_KGROUPS]):
            d.g[i] = L.KGroup(*g)
        d.n_aviews, d.n_groups = self.n_aviews, self.n_groups
        for k in ("b", "Ncols", "Ktot", "ldb", "W", "H", "NB", "bias", "rowvec", "rowvec_ld", "res", "res_dtype", "ldr",
                  "alpha", "accumulate", "out_f32", "ld_f32", "out_bf16", "ld_bf16", "act", "act_param", "split_off",
                  "block_n", "gn_stats", "stats_hw"):
            setattr(d, k, getattr(self, k) or 0)
        return d


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def desc_of(views, groups, weight, W, H, NB, *, bias=None, rowvec=None, res=None, alpha=1.0, accumulate=False,
            out_f32=None, out_bf16=None, act=L.ACT_NONE, act_param=0.0, split_off=0, block_n=0, ld_f32=None,
            ld_bf16=None, ldr=None, rowvec_ld=0, gn_stats=None, stats_hw=0, **_):
    """The descriptor tango_b200.lib.conv_gemm fills for these arguments."""
    return Desc(a=[(v.t.data_ptr() + 2 * v.off, v.C, v.W, v.H, v.NB, v.s_w, v.s_h, v.s_n) for v in views],
                g=[tuple(g) for g in groups], W=W, H=H, NB=NB, Ncols=weight.shape[0], Ktot=weight.shape[1],
                b=weight.data_ptr(), ldb=weight.stride(0), bias=_ptr(bias), rowvec=_ptr(rowvec), rowvec_ld=rowvec_ld,
                res=_ptr(res), res_dtype=(L.DT_BF16 if res is not None and res.element_size() == 2 else L.DT_F32),
                ldr=(res.stride(0) if ldr is None else ldr) if res is not None else 0, alpha=alpha,
                accumulate=int(accumulate), out_f32=_ptr(out_f32),
                ld_f32=(out_f32.stride(0) if ld_f32 is None else ld_f32) if out_f32 is not None else 0,
                out_bf16=_ptr(out_bf16),
                ld_bf16=(out_bf16.stride(0) if ld_bf16 is None else ld_bf16) if out_bf16 is not None else 0,
                act=act, act_param=act_param, split_off=split_off, block_n=block_n, gn_stats=_ptr(gn_stats),
                stats_hw=stats_hw if gn_stats is not None else 0)


def library_plan(d: Desc):
    """tng_gemm_plan of d: (block_n, M tile, ksplit), or None when it rejects d."""
    lib = L.load()
    bn, mode, ks = ctypes.c_int32(0), ctypes.c_int32(0), ctypes.c_int32(0)
    cd = d.ctypes()
    rc = lib.tng_gemm_plan(ctypes.byref(cd), ctypes.byref(bn), ctypes.byref(mode), ctypes.byref(ks))
    return None if rc != 0 else (bn.value, mode.value, ks.value)


# ---------------------------------------------------------------------------------------------------- the planner
@dataclass
class Plan:
    block_n: int
    bm: int
    ksplit: int
    fast_epi: bool
    stats: object          # None, "fused" or "after"
    bw: int
    bh: int
    bn: int
    tiles_w: int
    tiles_h: int
    tiles_n: int
    total_kiters: int
    ncols: int

    @property
    def key(self):
        return self.block_n, self.bm, self.ksplit

    @property
    def m_tiles(self):
        return self.tiles_w * self.tiles_h * self.tiles_n

    @property
    def n_tiles(self):
        return -(-self.ncols // self.block_n)

    @property
    def family(self):
        """The instantiation label tango_b200.lib's profiler gives the launch."""
        return f"gemm_tc<{self.block_n}" + (",splitk>" if self.ksplit > 1 else ",m256>" if self.bm == 256 else ">")


class Rejected(Exception):
    """TNG_EINVAL: what plan_gemm (or tng_conv_gemm before its launch) refuses."""


def _pow2(x):
    return x > 0 and x & (x - 1) == 0


def _f32(x):
    return struct.unpack("f", struct.pack("f", x))[0]


def tile_m(d, bm):
    """tile_m: the M box (bw, bh, bn) and the tile counts, or None when the grid does not allow the tiling."""
    if d.W >= bm or d.H == 1:
        bw, bh, bn = bm, 1, 1
    else:
        if not _pow2(d.W):
            return None
        bw, rem = d.W, bm // d.W
        if d.H >= rem:
            bh, bn = rem, 1
        else:
            if not _pow2(d.H):
                return None
            bh, bn = d.H, rem // d.H
    return dict(bm=bm, bw=bw, bh=bh, bn=bn, tiles_w=-(-d.W // bw), tiles_h=-(-d.H // bh), tiles_n=-(-d.NB // bn))


def full_m_tiles(d, t):
    if t["bh"] == 1 and t["bn"] == 1:
        return d.W % t["bw"] == 0
    return d.H % t["bh"] == 0 if t["bn"] == 1 else d.NB % t["bn"] == 0


def plan(d: Desc, sms: int) -> Plan:
    """plan_gemm at `sms` SMs; raises Rejected where it returns TNG_EINVAL."""
    geglu = d.act in GEGLU_ACTS
    if not 1 <= d.n_aviews <= L.MAX_AVIEWS:
        raise Rejected("n_aviews")
    if not 1 <= d.n_groups <= L.MAX_KGROUPS:
        raise Rejected("n_groups")
    if d.W <= 0 or d.H <= 0 or d.NB <= 0 or d.Ncols <= 0:
        raise Rejected("bad output grid")
    if (d.ldb if d.ldb > 0 else d.Ktot) % 8:
        raise Rejected("B row stride must be a multiple of 8 elements")
    t = tile_m(d, 128)
    if t is None:
        raise Rejected("W < 128 (and H when W * H < 128) must be a power of two")
    m_tiles = t["tiles_w"] * t["tiles_h"] * t["tiles_n"]
    bn_tile, ksplit = d.block_n, 1
    if geglu:
        if bn_tile == 0:
            bn_tile = 256 if d.Ncols % 256 == 0 else 128
        if bn_tile not in (128, 256) or d.Ncols % bn_tile or not d.out_bf16 or d.out_f32 or d.res or d.rowvec:
            raise Rejected("GEGLU epilogue needs block_n 128/256 dividing Ncols, bf16 output only")
        if _f32(d.alpha) != 1.0:
            raise Rejected("GEGLU epilogue needs alpha = 1")
    if bn_tile == 0:
        N = d.Ncols
        if N <= 32:
            bn_tile = 32
        elif N <= 64:
            bn_tile = 64
        elif N % 256 == 0 and m_tiles * (N // 256) >= 2 * sms:
            bn_tile = 256
        elif N % 160 == 0:
            bn_tile = 160
            if m_tiles * (N // 160) * 2 <= sms:      # under-filled launches
                kit = sum(g[5] for g in d.g[:d.n_groups])
                can_split = (d.out_f32 and not d.out_bf16 and not d.accumulate and d.act == L.ACT_NONE
                             and d.res != d.out_f32 and kit >= 32 and d.Ncols % 4 == 0)
                if can_split:
                    ksplit = 2
                elif N % 128 == 0 and m_tiles * (N // 128) <= sms:
                    bn_tile = 128
        elif N % 128 == 0:
            bn_tile = 128
        elif N % 64 == 0 and N < 256:
            bn_tile = 64
        else:
            bn_tile = 128
    total = 0
    for i, (view, a_c0, _dw, _dh, b_k0, nkb) in enumerate(d.g[:d.n_groups]):
        if view < 0 or view >= d.n_aviews or nkb <= 0:
            raise Rejected(f"k-group {i} invalid")
        if b_k0 < 0 or b_k0 + (nkb - 1) * BK >= d.Ktot:
            raise Rejected(f"k-group {i}: K block outside B")
        if a_c0 < 0 or a_c0 + (nkb - 1) * BK >= d.a[view][1]:
            raise Rejected(f"k-group {i}: K block outside view channels")
        total += nkb
    if not d.out_f32 and not d.out_bf16:
        raise Rejected("no output")
    if d.accumulate and not d.out_f32:
        raise Rejected("accumulate needs out_f32")
    al16 = lambda q: q % 16 == 0
    rowvec_ld = d.rowvec_ld if d.rowvec_ld > 0 else d.Ncols
    vec = not ((d.bias and not al16(d.bias))
               or (d.rowvec and (not al16(d.rowvec) or rowvec_ld % 4))
               or (d.res and (not al16(d.res) or (d.ldr % 8 if d.res_dtype == L.DT_BF16 else d.ldr % 4)))
               or (d.out_f32 and (not al16(d.out_f32) or d.ld_f32 % 4))
               or (d.out_bf16 and (not al16(d.out_bf16) or d.ld_bf16 % 8 or d.split_off % 8)))
    fast_epi = vec and d.Ncols % 4 == 0
    if geglu and not vec:
        raise Rejected("GEGLU epilogue needs 16-byte aligned output")
    if d.gn_stats:
        if d.stats_hw <= 0 or (d.W * d.H * d.NB) % d.stats_hw:
            raise Rejected("gn_stats: the output rows must be whole images of stats_hw pixels")
        if not d.out_f32 and (d.split_off > 0 or d.act != L.ACT_NONE):
            raise Rejected("gn_stats without an fp32 output needs a plain bf16 output")
    if ksplit > 1 and not fast_epi:
        ksplit = 1
    n_tiles = -(-d.Ncols // bn_tile)
    if bn_tile == 160 and ksplit == 1 and fast_epi and total >= 64 and not geglu:
        q = tile_m(d, 256)
        if q is not None and 2 * q["tiles_w"] * q["tiles_h"] * q["tiles_n"] * n_tiles >= sms and \
                (not d.gn_stats or full_m_tiles(d, q)):
            t = q
    stats = None
    if d.gn_stats:
        fused = (full_m_tiles(d, t) and d.Ncols % bn_tile == 0 and fast_epi and ksplit == 1 and not d.accumulate
                 and d.stats_hw % 16 == 0 and not geglu)
        stats = "fused" if fused else "after"
        stored, ld = (d.out_f32, d.ld_f32) if d.out_f32 else (d.out_bf16, d.ld_bf16)
        if stats == "after" and (d.Ncols % 4 or ld % 4 or stored % 8):
            raise Rejected("gn_stats after the GEMM needs Ncols % 4 == 0 and an 8-byte aligned output with ld % 4 == 0")
    return Plan(block_n=bn_tile, bm=t["bm"], ksplit=ksplit, fast_epi=bool(fast_epi), stats=stats, bw=t["bw"], bh=t["bh"],
             bn=t["bn"], tiles_w=t["tiles_w"], tiles_h=t["tiles_h"], tiles_n=t["tiles_n"], total_kiters=total,
             ncols=d.Ncols)
    return p


def launch_check(d: Desc, p: Plan) -> None:
    """What tng_conv_gemm refuses after planning: a view whose C is not a multiple of 8 (each of the four tensor maps
    is encoded, unused ones from view 0), an N tile without a kernel."""
    for i in range(4):
        if d.a[i if i < d.n_aviews else 0][1] % 8:
            raise Rejected(f"view {i}: C must be a multiple of 8")
    if p.block_n not in BNS:
        raise Rejected(f"block_n={p.block_n} unsupported")


# ---------------------------------------------------------------------------------------------------- the dispatch
def _body(d, p, nvalid, full, mode):
    if d.act in GEGLU_ACTS:
        if d.act == L.ACT_GEGLU_TANH:
            return "GEGLU:tanh-hilo" if d.split_off > 0 else "GEGLU:tanh"
        if d.split_off > 0:
            return "GEGLU:erf-hilo"
        return "GEGLU:erf-full" if nvalid == p.bm else "GEGLU:erf-partial"
    if full:
        return f"FULL:{mode}"
    return "VEC" if p.fast_epi else "SCALAR"


def _features(d, p, body, sp, mode):
    if body.startswith("GEGLU"):
        return ["run"]
    f = ["run"]
    add_terms = p.ksplit == 1 or sp == 0
    if d.rowvec and add_terms:
        f.append("rowvec:warp" if (p.bw * p.bh) % 16 == 0 else "rowvec:slot")
    if d.out_f32 and d.accumulate:
        f.append("accumulate")
    if d.out_bf16:
        if d.act == L.ACT_SILU:
            f.append("act:silu")
        elif d.act == L.ACT_LRELU:
            f.append("act:lrelu")
        if d.split_off > 0:
            f.append("hilo")
    if not body.startswith("FULL"):
        f.append(f"mode:{mode}")
    if p.ksplit > 1:
        f.append("red:odd" if p.total_kiters % 2 else "red:even")
    if p.stats == "fused" and body.startswith("FULL"):
        f.append("stats:fused")
    elif p.stats == "after":
        f.append("stats:after")
    return f


def work_items(d: Desc, p: Plan, sms: int):
    """(CTA, body, features) of every work item, in each CTA's order (gemm_tc_kernel: work_item, nvalid, full)."""
    mode = (1 if d.res else 0) | (2 if d.out_f32 else 0) | (4 if d.out_bf16 else 0)
    n_tiles = p.n_tiles
    work = p.m_tiles * n_tiles * p.ksplit
    grid = min(work, sms)
    for tile in range(work):
        sp, t2 = tile % p.ksplit, tile // p.ksplit
        tm, tn = t2 // n_tiles, t2 % n_tiles
        tw, th, tb = tm % p.tiles_w, (tm // p.tiles_w) % p.tiles_h, tm // (p.tiles_w * p.tiles_h)
        w0, h0, n0 = tw * p.bw, th * p.bh, tb * p.bn
        if p.bh == 1 and p.bn == 1:
            nvalid = min(p.bm, d.W - w0)
        elif p.bn == 1:
            nvalid = min(p.bh, d.H - h0) * p.bw
        else:
            nvalid = min(p.bn, d.NB - n0) * p.bh * p.bw
        full = p.fast_epi and p.ksplit == 1 and nvalid == p.bm and (tn + 1) * p.block_n <= d.Ncols
        body = _body(d, p, nvalid, full, mode)
        yield tile % grid, body, _features(d, p, body, sp, mode)


def cells(d: Desc, sms: int, p: Plan = None) -> set:
    """The (BN, BM, body, feature) cells a launch of d runs at `sms` SMs (raises Rejected where tng_conv_gemm fails)."""
    p = plan(d, sms) if p is None else p
    launch_check(d, p)
    out, ran_full = set(), set()
    for cta, body, feats in work_items(d, p, sms):
        if body.startswith("FULL") or body == "GEGLU:erf-full":
            ran_full.add(cta)
        elif cta in ran_full and body in ("VEC", "GEGLU:erf-partial"):
            feats = feats + ["after-full"]
        out.update((p.block_n, p.bm, body, f) for f in feats)
    return out


# ---------------------------------------------------------------------------------------------------- the matrix
def _exclusion(bn, bm, body, f):
    """Why the dispatch cannot reach cell (bn, bm, body, f), or None when it can."""
    if bm == 256 and bn != 160:
        return "256-row tiles are planned for block_n 160 only"
    if body.startswith("GEGLU"):
        if (bn, bm) not in ((128, 128), (256, 128)):
            return "GEGLU is planned on 128-row tiles with block_n 128 or 256 only"
        if f == "after-full":
            return None if body == "GEGLU:erf-partial" else "this GEGLU body does not depend on the tile being full"
        if f != "run":
            return "GEGLU takes no row vector, residual, fp32 output or statistics; its activation and hi/lo are the body"
        return None
    if body == "SCALAR" and bm == 256:
        return "256-row tiles need fast_epi (16-byte aligned epilogue operands)"
    full = body.startswith("FULL")
    mode = int(body[5:]) if full else None
    if f == "after-full":
        return None if body == "VEC" else ("FULL bodies are the full tiles" if full else
                                           "a launch without fast_epi runs no FULL tile")
    if f.startswith("mode:") and full:
        return "a FULL body fixes its mode at compile time"
    if f == "accumulate" and full and not mode & 2:
        return "accumulate needs an fp32 output"
    if f in ("act:silu", "act:lrelu", "hilo") and full and not mode & 4:
        return "the activation and the hi/lo split act on the bf16 output only"
    if f.startswith("red:"):
        if body != "VEC":
            return "split-K tiles take the VEC body"
        if (bn, bm) != (160, 128):
            return "split-K is planned on the automatic block_n 160 path with 128-row tiles only"
    if f == "stats:fused" and not full:
        return "fused statistics need every tile full: FULL bodies only"
    if f == "stats:after" and body == "VEC" and bm == 256:
        return "256-row tiles with statistics are planned only when every tile is full (block_n 160 divides Ncols)"
    return None


ALL_CELLS = [(bn, bm, body, f) for bn in BNS for bm in BMS for body in BODIES for f in FEATURES]
EXCLUDED = {c: r for c in ALL_CELLS if (r := _exclusion(*c)) is not None}
REACHABLE = frozenset(c for c in ALL_CELLS if c not in EXCLUDED)


def matrix(covered, *, only=None) -> str:
    """The covered cells as a table: one row per (BN, BM, body), one column per feature ('x' covered, '.' reachable and
    not covered, blank unreachable)."""
    cols = [f.replace("rowvec:", "rv:").replace("stats:", "st:").replace("mode:", "m") for f in FEATURES]
    lines = [f"{'BN x BM  body':<27s} " + " ".join(f"{c:>5s}" for c in cols)]
    for bn, bm in INSTANTIATIONS:
        for body in BODIES:
            row = [(bn, bm, body, f) for f in FEATURES]
            if not any(c in REACHABLE for c in row):
                continue
            marks = ["x" if c in covered else "." if c in REACHABLE else " " for c in row]
            lines.append(f"{bn:>3d} x {bm:<3d} {body:<18s} " + " ".join(f"{m:>5s}" for m in marks))
    return "\n".join(lines)
