"""GPU: every kernel launch of production-size generations checked against its contract with its own descriptor,
buffers and inputs (tests/launch_audit.py). The models are the Tango base architecture with seeded random weights and
a FLAN-T5-large text encoder, CUDA graphs off (each launch runs eagerly, so the audit sees it), seeded inputs:

  bench     bf16, 8 prompts of mixed length under CFG (UNet batch 16), 2 DDPM steps at 256 x 16, decode + vocoder
  parity    split, the same prompts, 1 step, decode + vocoder
  30 s      bf16, 8 prompts at 768 x 16 (the elementwise walks exceed grid_for's cap), 1 step, decode of 2 latents
  samplers  bf16, 3 steps each of DPM-Solver++ (order 3) and UniPC: the latent-step entry points
  edit      bf16 inpainting edit of two 163 872-sample clips, 2 steps

Each run also checks its own premises (the plan families and epilogue paths it claims to cover, the walk lengths, the
launch count of a forward against a graph-captured one), so that a planning change fails here instead of quietly
shrinking what is covered."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from launch_audit import LATENT_STEPS, install_audit
from tango_b200 import lib as L
from tango_b200 import synth
from tango_b200.pipeline import Tango
from tango_b200.schedulers import DPMSolverMultistepScheduler, UniPCMultistepScheduler

pytestmark = pytest.mark.gpu

PROMPTS = ["a dog barks", "rain falling on a tin roof while thunder rolls in the distance",
           "a man speaks", "an orchestra tunes up before a concert, then the audience applauds politely",
           "birds chirp", "a car engine starts, idles for a while and then drives away down a gravel road",
           "waves crash on the shore", "church bells ring"]
GUIDANCE = 3.0


def num_sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_cap_threads() -> int:
    return num_sms() * 16 * 256          # grid_for: at most 16 CTAs of 256 threads per SM


def build(cuda, precision):
    t = Tango.from_synthetic(device=cuda, precision=precision, t5_config=synth.FLAN_T5_LARGE_CONFIG)
    t.model.use_cuda_graph = False       # also the decode (Tango._decode follows the model's flag)
    t.model._ensure_text_encoder()
    t.model.text_encoder.use_cuda_graph = False
    return t


@pytest.fixture(scope="module")
def bf16_model(cuda):
    t = build(cuda, "bf16")
    yield t
    del t
    torch.cuda.empty_cache()


def count_forwards(monkeypatch, unet, audit):
    """Wrap unet.forward_rows: per forward, (library launches, launches that went through an audited wrapper)."""
    fw, counts = unet.forward_rows, []

    def counted(*a, **k):
        n0, r0 = L.launch_count(), sum(r.launches for r in audit.records)
        out = fw(*a, **k)
        counts.append((L.launch_count() - n0, sum(r.launches for r in audit.records) - r0))
        return out

    monkeypatch.setattr(unet, "forward_rows", counted)
    return counts


def graph_launches_per_forward(t, latent_shape):
    """launches_per_forward of a graph-captured forward of the same shape (one step, outside the audit)."""
    m = t.model
    m.use_cuda_graph = True
    try:
        m.inference(PROMPTS, t.scheduler, 1, GUIDANCE, generator=torch.Generator(device=t.device).manual_seed(1),
                    latent_shape=latent_shape)
        n = m.launches_per_forward
    finally:
        m.use_cuda_graph = False
        m._invalidate()
    assert n > 0
    return n


def report(audit, title):
    print()
    print(audit.table(title))
    assert audit.audited() == set(audit.calls), "an entry point the run used was never audited"


def test_bench_configuration(cuda, bf16_model, monkeypatch):
    t = bf16_model
    lpf = graph_launches_per_forward(t, (256, 16))
    audit = install_audit(monkeypatch)
    counts = count_forwards(monkeypatch, t.model.unet, audit)
    g = torch.Generator(device=cuda).manual_seed(1234)
    waves = t.generate_for_batch(PROMPTS, steps=2, guidance=GUIDANCE, batch_size=8, generator=g,
                                 latent_shape=(256, 16))
    report(audit, "bench: bf16, 8 prompts, CFG, 2 DDPM steps, 256 x 16, decode + vocoder")
    assert len(waves) == 8 and waves[0].shape == (163872,)
    fams, tags = {r.family for r in audit.records}, audit.tags()
    assert "gemm_tc<160,m256>" in fams, sorted(fams)
    assert any("splitk" in f for f in fams), sorted(fams)
    assert {"geglu", "stats-fused", "stats-after"} <= tags, tags
    assert len(counts) == 2 and all(c == (lpf, lpf) for c in counts), (counts, lpf)


def test_parity_configuration(cuda, monkeypatch):
    t = build(cuda, "split")
    audit = install_audit(monkeypatch)
    g = torch.Generator(device=cuda).manual_seed(1234)
    t.generate_for_batch(PROMPTS, steps=1, guidance=GUIDANCE, batch_size=8, generator=g, latent_shape=(256, 16))
    report(audit, "parity: split, 8 prompts, CFG, 1 DDPM step, 256 x 16, decode + vocoder")
    assert any(r.entry == "attention" and "hi/lo" in r.shape for r in audit.records)
    assert {"softmax_rows", "transpose_bf16"} <= audit.audited()      # the split-mode VAE attention
    del t
    torch.cuda.empty_cache()


def test_30s_configuration(cuda, bf16_model, monkeypatch):
    t = bf16_model
    lpf = graph_launches_per_forward(t, (768, 16))
    audit = install_audit(monkeypatch)
    counts = count_forwards(monkeypatch, t.model.unet, audit)
    g = torch.Generator(device=cuda).manual_seed(4321)
    with torch.no_grad():
        lat = t.model.inference(PROMPTS, t.scheduler, 1, GUIDANCE, generator=g, latent_shape=(768, 16))
        waves = t._decode(lat[:2])
    report(audit, "30 s: bf16, 8 prompts, CFG, 1 DDPM step, 768 x 16, decode of 2")
    assert waves.shape == (2, 4 * 768 * 160 + 32)
    cap = grid_cap_threads()
    assert any(r.entry in LATENT_STEPS and r.work > cap for r in audit.records)
    assert any(r.entry == "cast_act" and r.work > 4 * cap for r in audit.records)   # several 4-iteration batches
    assert any(r.entry == "attention_wide" and r.shape.split("x")[1] == "12288" for r in audit.records)
    assert counts == [(lpf, lpf)], (counts, lpf)


@pytest.mark.parametrize("sampler", ["dpmsolver++", "unipc"])
def test_sampler_latent_steps(cuda, bf16_model, monkeypatch, sampler):
    t = bf16_model
    if sampler == "dpmsolver++":
        sch = DPMSolverMultistepScheduler.from_config(t.scheduler.config, solver_order=3, lower_order_final=False)
    else:
        sch = UniPCMultistepScheduler.from_config(t.scheduler.config, solver_order=3, lower_order_final=False)
    audit = install_audit(monkeypatch, only=LATENT_STEPS)
    g = torch.Generator(device=cuda).manual_seed(77)
    with torch.no_grad():
        t.model.inference(PROMPTS, sch, 3, GUIDANCE, generator=g, latent_shape=(256, 16))
    print()
    print(audit.table(f"samplers: {sampler}, bf16, 8 prompts, 3 steps"))
    entry = "dpm_step" if sampler == "dpmsolver++" else "unipc_step"
    assert sum(r.entry == entry for r in audit.records) == 3
    assert audit.audited() == set(audit.calls) & set(LATENT_STEPS)


def test_edit_configuration(cuda, bf16_model, monkeypatch):
    t = bf16_model
    rng = np.random.default_rng(5)
    clips = [(0.3 * rng.standard_normal(163872)).astype(np.float32) for _ in range(2)]
    audit = install_audit(monkeypatch)
    g = torch.Generator(device=cuda).manual_seed(99)
    waves = t.edit_for_batch(PROMPTS[:2], clips, strength=1.0, steps=2, guidance=GUIDANCE, batch_size=2, generator=g,
                             time_mask_ratio_start_and_end=(0.25, 0.75))
    report(audit, "edit: bf16 inpainting, 2 prompts, 163 872-sample clips, 2 steps")
    assert len(waves) == 2
    assert {"stft_frames", "stft_magnitude", "log_clamp", "latent_blend"} <= audit.audited()
