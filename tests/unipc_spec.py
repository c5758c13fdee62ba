"""Executable statement of what `tng_unipc_step` computes (TEST INFRASTRUCTURE ONLY).

The UniPC counterpart of the latent-update statements in cabi_spec.py: the same contract as include/tango_b200.h in
torch on the CPU, one op per kernel op in the same association, so that the scheduler's host code (coefficient rows,
orders, history slots, the corrected-sample buffer) can be checked without a GPU and the kernel can be checked against
it on one. `install_unipc_spec_backend` adds it to cabi_spec's spec backend. It is never imported by the package.
"""
from __future__ import annotations

import torch

from cabi_spec import _guided_output, _pack_next_in, install_spec_backend
from oracle.unipc import fma32


def spec_unipc_step(model_out, cfg, guidance, sample, coef, corrector_order, predictor_order, m_cur, m_prev, last, prev,
                    next_in, *, B, Cc, HW, split_off=0):
    """CFG combine + conversion to m_cur + UniC corrector of corrector_order (0: none) from last (overwritten with the
    corrected sample) + UniP predictor of predictor_order from the history slots m_prev = (m_{i-1}, ...) + packing."""
    c = [coef.reshape(-1)[i] for i in range(18)]
    s = sample.reshape(B, Cc, HW).float()
    v = _guided_output(model_out, cfg, guidance, B=B, Cc=Cc, HW=HW)
    m = (c[0] * s + c[1] * v) / c[2]
    m_cur.reshape(B, Cc, HW).copy_(m)
    h = [t.reshape(B, Cc, HW) for t in m_prev]
    p, q = corrector_order, predictor_order
    x = s
    if p > 0:
        corr = torch.zeros_like(m)
        if p >= 2:
            corr = c[8] * ((h[1] - h[0]) / c[6])
        if p == 3:
            corr = fma32(c[9].expand_as(m), (h[2] - h[0]) / c[7], corr)
        x = (c[3] * last.reshape(B, Cc, HW) - c[4] * h[0]) - c[5] * (corr + c[10] * (m - h[0]))
    if last is not None:
        last.reshape(B, Cc, HW).copy_(x)
    res = torch.zeros_like(m)
    if q >= 2:
        res = c[16] * ((h[0] - m) / c[14])
    if q == 3:
        res = fma32(c[17].expand_as(m), (h[1] - m) / c[15], res)
    out = (c[11] * x - c[12] * m) - c[13] * res
    if prev is not None:
        prev.reshape(B, Cc, HW).copy_(out)
    _pack_next_in(next_in, out, cfg, split_off, B=B, Cc=Cc, HW=HW)


def install_unipc_spec_backend(monkeypatch):
    """cabi_spec's spec backend plus tango_b200.lib.unipc_step as its statement (under pytest's monkeypatch only)."""
    from tango_b200 import lib as L
    install_spec_backend(monkeypatch)
    monkeypatch.setattr(L, "unipc_step", spec_unipc_step)
