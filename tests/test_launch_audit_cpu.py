"""CPU: the launch audit (tests/launch_audit.py) over the spec backend. Every launch of a tiny UNet forward, a tiny
decode and a tiny T5 encode, with the statements of cabi_spec.py standing in for the kernels, must meet its contract;
and a statement perturbed in one line (a column off by 1e-3, a stray write, an unwritten row, statistics missing a row)
must fail the audit at the launch it corrupts."""
import os

import numpy as np
import pytest
import torch

import cabi_spec as S
from launch_audit import SPECS, AuditFailure, install_audit
from tango_b200 import lib as L
from tango_b200 import synth
from tango_b200.t5 import T5EncoderModel
from tango_b200.unet import UNet2DConditionModel
from unipc_spec import install_unipc_spec_backend

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CPU = torch.device("cpu")


@pytest.fixture(autouse=True)
def _spec_backend(monkeypatch):
    install_unipc_spec_backend(monkeypatch)


def tiny_unet_forward(precision):
    gd = np.load(os.path.join(GOLD, "tiny_unet.npz"))
    cfg = synth.TINY_UNET_CONFIG
    u = UNet2DConditionModel.from_config(cfg, precision=precision).to(CPU)
    u.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    return u(torch.from_numpy(gd["sample"]), torch.tensor(int(gd["t"])), torch.from_numpy(gd["ehs"]),
             encoder_attention_mask=torch.from_numpy(gd["mask"])).sample


def tiny_decode(precision):
    from tango_b200.vae import AutoencoderKL
    gd = np.load(os.path.join(GOLD, "tiny_vae_vocoder.npz"))
    vae = AutoencoderKL(**synth.VAE_CONFIG, precision=precision).to(CPU)
    vae.load_state_dict(synth.synth_state_dict(synth.vae_decoder_param_shapes(), seed=0))
    return vae.decode_to_waveform(vae.decode_first_stage(torch.from_numpy(gd["z"])))


def tiny_t5_encode(precision):
    gd = np.load(os.path.join(GOLD, "tiny_t5.npz"))
    cfg = synth.TINY_T5_CONFIG
    m = T5EncoderModel.from_config(cfg, precision=precision).to(CPU)
    m.load_state_dict(synth.synth_state_dict(synth.t5_encoder_param_shapes(cfg), seed=0))
    return m(torch.from_numpy(gd["ids_long"]), torch.from_numpy(gd["mask_long"]))[0]


RUNS = {"unet": tiny_unet_forward, "decode": tiny_decode, "t5": tiny_t5_encode}


@pytest.mark.parametrize("precision", ["bf16", "split"])
@pytest.mark.parametrize("run", sorted(RUNS))
def test_spec_backend_meets_every_contract(monkeypatch, run, precision):
    audit = install_audit(monkeypatch)
    RUNS[run](precision)
    assert audit.records and all(r.excess <= 1.0 for r in audit.records)
    assert audit.audited() == set(audit.calls)
    print(audit.table(f"tiny {run} ({precision})"))


def test_only_passes_other_launches_through(monkeypatch):
    audit = install_audit(monkeypatch, only=["layernorm"])
    tiny_unet_forward("bf16")
    assert audit.audited() == {"layernorm"} and audit.calls["conv_gemm"] > 0
    assert len(audit.records) == audit.calls["layernorm"]


# ---------------------------------------------------------------------------------------------------- perturbations
def _first_f32_gemm(spec):
    """spec_conv_gemm, perturbed by `spec(kw)` after it ran, on the first launch with an fp32 output only."""
    seen = []

    def conv_gemm(views, groups, weight, W, H, NB, **kw):
        S.spec_conv_gemm(views, groups, weight, W, H, NB, **kw)
        if kw.get("out_f32") is not None and not seen:
            seen.append(1)
            spec(weight, W * H * NB, kw)
    return conv_gemm


def column_off(weight, rows, kw):
    kw["out_f32"][:, 3] *= 1.0 + 1e-3


def write_past_ncols(weight, rows, kw):
    o = kw["out_f32"]
    o.as_strided((1,), (1,), o.storage_offset() + weight.shape[0]).fill_(1234.5)


def stats_missing_a_row(weight, rows, kw):
    if kw.get("gn_stats") is None:
        raise AssertionError("the first fp32 GEMM of the tiny UNet carries GroupNorm statistics")
    y = kw["out_f32"][0, :weight.shape[0]].double()
    kw["gn_stats"][0, :, 0] -= y
    kw["gn_stats"][0, :, 1] -= y * y


def unwritten_row(x0, st0, x1, st1, NB, HW, groups, gamma, beta, eps, act, y, **kw):
    keep = y[5].clone()
    S.spec_groupnorm(x0, st0, x1, st1, NB, HW, groups, gamma, beta, eps, act, y, **kw)
    y[5] = keep


PERTURBED = {"one conv_gemm column off by 1e-3": ("conv_gemm", _first_f32_gemm(column_off)),
             "conv_gemm writes one column past Ncols": ("conv_gemm", _first_f32_gemm(write_past_ncols)),
             "gn_stats missing one row": ("conv_gemm", _first_f32_gemm(stats_missing_a_row)),
             "groupnorm leaves a row unwritten": ("groupnorm", unwritten_row)}


@pytest.mark.parametrize("case", sorted(PERTURBED))
def test_perturbed_statement_fails_at_its_launch(monkeypatch, case):
    entry, fn = PERTURBED[case]
    monkeypatch.setattr(L, entry, fn)
    audit = install_audit(monkeypatch)
    with pytest.raises(AuditFailure, match=rf"launch #\d+ {entry} "):
        tiny_unet_forward("bf16")
    assert all(r.excess <= 1.0 for r in audit.records)     # every launch before it passed


def test_every_entry_point_has_a_check():
    from launch_audit import CHECKS, EXACT, REGIONS
    assert set(SPECS) == set(REGIONS) == set(CHECKS) | set(EXACT)
    assert "unipc_step" in SPECS
