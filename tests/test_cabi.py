"""CPU: libtango_b200.so loads without a GPU and exports every symbol include/tango_b200.h declares."""
import ctypes
import os
import re

import torch

from tango_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "tango_b200.h")).read()
    return sorted(set(re.findall(r"\b(tng_[a-z0-9_]+)\s*\(", src)))


def test_exports_match_header():
    lib = L.load()
    names = header_symbols()
    assert len(names) >= 16
    for n in names:
        assert hasattr(lib, n), f"{n} not exported"
    assert sorted(L.SYMBOLS) == names
    assert lib.tng_version() >= 100


def test_struct_sizes_match_c_layout():
    # tng_aview: ptr + 7 x int64; tng_kgroup: 6 x int32
    assert ctypes.sizeof(L.AView) == 64 and ctypes.sizeof(L.KGroup) == 24
    assert ctypes.sizeof(L.GemmDesc) % 8 == 0


def test_compute_call_fails_loudly_without_gpu():
    if torch.cuda.is_available():
        return
    lib = L.load()
    d = L.GemmDesc()
    d.n_aviews, d.n_groups, d.W, d.H, d.NB, d.Ncols, d.Ktot = 1, 1, 128, 1, 1, 64, 64
    d.g[0] = L.KGroup(0, 0, 0, 0, 0, 1)
    d.a[0] = L.AView(0, 64, 128, 1, 1, 64, 8192, 8192)
    buf = ctypes.create_string_buffer(64)
    d.out_f32 = ctypes.addressof(buf)
    d.ld_f32 = 64
    rc = lib.tng_conv_gemm(ctypes.byref(d), None)
    assert rc != 0 and len(lib.tng_last_error()) > 0


def _geglu_desc(buf, **kw):
    """A valid GEGLU descriptor (2 N tiles of 256, bf16 output) over host memory: tng_gemm_plan never touches it."""
    base = (ctypes.addressof(buf) + 255) // 256 * 256
    d = L.GemmDesc()
    d.n_aviews, d.n_groups, d.W, d.H, d.NB, d.Ncols, d.Ktot = 1, 1, 300, 1, 1, 512, 64
    d.g[0] = L.KGroup(0, 0, 0, 0, 0, 1)
    d.a[0] = L.AView(base, 64, 300, 1, 1, 64, 64 * 300, 64 * 300)
    d.b, d.out_bf16, d.ld_bf16, d.act, d.alpha = base, base, 256, L.ACT_GEGLU, 1.0
    for k, v in kw.items():
        setattr(d, k, base if v is True else v)
    return d


def test_gemm_plan_rejects_unsupported_geglu_epilogues():
    """The GEGLU epilogue applies the bias only: tng_gemm_plan (and so tng_conv_gemm) refuses alpha != 1, as it refuses a
    residual, a row vector or an fp32 output; no device is needed to plan."""
    lib = L.load()
    buf = ctypes.create_string_buffer(1 << 16)
    bn = ctypes.c_int32(0)
    plan = lambda d: lib.tng_gemm_plan(ctypes.byref(d), ctypes.byref(bn), None, None)
    for act in (L.ACT_GEGLU, L.ACT_GEGLU_TANH):
        assert plan(_geglu_desc(buf, act=act)) == 0 and bn.value == 256
        for bad in (dict(alpha=0.5), dict(alpha=3.0), dict(alpha=-1.0), dict(res=True, ldr=512), dict(rowvec=True),
                    dict(out_f32=True, ld_f32=512), dict(block_n=64)):
            assert plan(_geglu_desc(buf, act=act, **bad)) == -1, bad
            assert b"GEGLU" in lib.tng_last_error()


def test_linear_f32_rejects_activations_other_than_none_and_silu():
    """tng_linear_f32 applies NONE or SILU only: every other activation id is TNG_EINVAL before any launch (LRELU would
    run with a slope of 0, GEGLU as the identity)."""
    lib = L.load()
    x, w, y = (ctypes.create_string_buffer(4 * 64) for _ in range(3))
    for pre, post in ((L.ACT_LRELU, L.ACT_NONE), (L.ACT_NONE, L.ACT_LRELU), (L.ACT_GEGLU, L.ACT_NONE),
                      (L.ACT_NONE, L.ACT_GEGLU_TANH), (L.ACT_SILU, 5), (-1, L.ACT_SILU)):
        rc = lib.tng_linear_f32(ctypes.addressof(x), 2, 8, ctypes.addressof(w), None, 4, pre, post, ctypes.addressof(y),
                                None)
        assert rc == -1 and b"linear_f32" in lib.tng_last_error(), (pre, post)


def test_latent_updates_reject_bad_arguments_before_any_launch():
    """tng_sched_step, tng_dpm_step and tng_latent_blend share their checks: required pointers, B, C and HW >= 1,
    ld_mo >= C, split_off 0 or >= C and ld_in >= C + split_off, plus each entry point's own. Every failure is TNG_EINVAL
    naming the entry point, returned before any CUDA call, so host buffers and no device suffice."""
    lib = L.load()
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    C = 4
    common = dict(coef=p, next_in=p, ld_in=2 * C, split_off=C, cfg=1, B=2, C=C, HW=8, stream=None)
    calls = {
        "sched_step": (lib.tng_sched_step, "model_out ld_mo cfg guidance sample noise coef prev next_in ld_in "
                       "split_off B C HW stream", dict(model_out=p, ld_mo=C, guidance=3.0, sample=p, noise=p, prev=p),
                       ["sample", "coef"]),
        "dpm_step": (lib.tng_dpm_step, "model_out ld_mo cfg guidance sample coef order m0 m1 m2 prev next_in ld_in "
                     "split_off B C HW stream", dict(model_out=p, ld_mo=C, guidance=3.0, sample=p, order=3, m0=p, m1=p,
                                                     m2=p, prev=p), ["model_out", "sample", "coef", "m0"]),
        "latent_blend": (lib.tng_latent_blend, "x0 noise mask mask_bstride coef sample next_in ld_in cfg split_off B C "
                         "HW stream", dict(x0=p, noise=p, mask=p, mask_bstride=8, sample=p), ["x0", "coef", "sample"]),
    }
    for name, (fn, argnames, own, required) in calls.items():
        good = dict(common, **own)
        bad = [{k: None} for k in required]
        bad += [dict(B=0), dict(C=0), dict(HW=0), dict(B=-1), dict(split_off=1), dict(split_off=C - 1),
                dict(split_off=-C), dict(ld_in=2 * C - 1), dict(split_off=0, ld_in=C - 1)]
        if "ld_mo" in good:
            bad += [dict(ld_mo=C - 1), dict(ld_mo=0), dict(prev=None, next_in=None)]
        if name == "dpm_step":
            bad += [dict(order=0), dict(order=4), dict(m1=None), dict(order=2, m1=None), dict(m2=None)]
        if name == "latent_blend":
            bad.append(dict(mask_bstride=-1))
        for change in bad:
            args = {**good, **change}
            rc = fn(*[args[a] for a in argnames.split()])
            assert rc == -1 and name.encode() in lib.tng_last_error(), (name, change, rc, lib.tng_last_error())
