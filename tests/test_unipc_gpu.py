"""GPU: the multistep UniPC scheduler on tng_unipc_step, against the fork's scheduler run through the unmodified reference
(tests/golden/unipc.npz, oracle/make_golden_unipc.py): `step` bit for bit over every golden loop, the tiny CFG loop,
the tiny edit and inpaint loops, config 1 at full size at 10 steps, the prompt-sharded batch path and the kernel's
C-ABI edges."""
import json
import os

import numpy as np
import pytest
import torch

from unipc_spec import spec_unipc_step
from oracle import edit as oedit
from oracle import make_golden_config1 as c1
from tango_b200 import lib as L
from tango_b200 import parallel, synth
from tango_b200.pipeline import AudioDiffusion, Tango
from tango_b200.schedulers import DDPMScheduler, UniPCMultistepScheduler

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def unipc(**kw):
    return UniPCMultistepScheduler.from_config(DDPMScheduler.from_pretrained().config, **kw)


def test_step_bit_exact_over_every_golden_loop(cuda):
    gd = np.load(os.path.join(GOLD, "unipc.npz"))
    n = 4 * 3 * 8 * 8
    x_fork = (torch.arange(n).reshape(3, 8, 8, 4) / n).permute(3, 0, 1, 2).contiguous()
    for k, (kw, steps, model) in enumerate(json.loads(str(gd["loop_configs"]))):
        s = UniPCMultistepScheduler(**kw)
        s.set_timesteps(steps, device=cuda)
        x = (torch.from_numpy(gd["sin_x0"]) if model == "sin" else x_fork).to(cuda)
        for t in s.timesteps:
            xc, tc = x.cpu(), t.cpu()     # the model is evaluated on the CPU, as in the golden generator
            mo = torch.sin(xc * 3.0 + float(tc) / 1000) if model == "sin" else xc * tc / (tc + 1)
            x = s.step(mo.to(cuda), t, x).prev_sample
        assert np.array_equal(x.cpu().numpy(), gd[f"loop_{k}"]), f"loop {k} {kw} {steps} steps not bit-exact"


def tiny_model(cuda, precision, **kw):
    cfg = synth.TINY_UNET_CONFIG
    m = AudioDiffusion(unet_config=cfg, precision=precision, **kw).to(cuda)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    return m


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_tiny_inference_vs_golden(cuda, precision):
    gd, ti = np.load(os.path.join(GOLD, "unipc.npz")), np.load(os.path.join(GOLD, "tiny_inference.npz"))
    kw = dict(prompt_embeds=torch.from_numpy(ti["embeds"]), boolean_prompt_mask=torch.from_numpy(ti["mask"]),
              latents=torch.from_numpy(ti["lat0"]), latent_shape=(32, 16))
    m = tiny_model(cuda, precision)
    lat = m.inference(["synthetic prompt"], unipc(), 6, 3.0, **kw).clone()
    e = rel(lat, gd["tiny_latents"])
    print(f"tiny 6-step UniPC-2 bh2 CFG loop {precision}: rel err vs reference golden {e:.3e}")
    assert e < (1e-3 if precision == "split" else 6e-2)
    # a second call on the same shape reuses the graph, the history slots and the corrected-sample buffer
    again = m.inference(["synthetic prompt"], unipc(), 6, 3.0, **kw)
    assert rel(again, lat) < (1e-4 if precision == "split" else 6e-2)
    lat2 = tiny_model(cuda, precision, use_cuda_graph=False).inference(["synthetic prompt"], unipc(), 6, 3.0, **kw)
    assert rel(lat, lat2) < (1e-4 if precision == "split" else 6e-2)


@pytest.mark.parametrize("case", ["tiny_unipc", "tiny_unipc_inpaint"])
def test_tiny_edit_vs_golden(cuda, case):
    gd, ti = np.load(os.path.join(GOLD, "unipc.npz")), np.load(os.path.join(GOLD, "tiny_inference.npz"))
    c = json.loads(str(gd["edit_cases"]))[case]
    x0 = torch.from_numpy(gd[f"{case}_x0"])
    noise = oedit.seeded_draws(c["seed"], tuple(x0.shape), 0)[1]
    mask = torch.from_numpy(gd[f"{case}_mask"]) if f"{case}_mask" in gd else None
    lat = tiny_model(cuda, "split").inference(
        None, unipc(), c["steps"], c["guidance"], prompt_embeds=torch.from_numpy(ti["embeds"]),
        boolean_prompt_mask=torch.from_numpy(ti["mask"]), latent_shape=tuple(c["latent_shape"]), init_latents=x0,
        init_noise=noise, strength=c["strength"], inpaint_mask=mask)
    e = rel(lat, gd[f"{case}_latents"])
    print(f"{case}: rel err vs reference golden {e:.3e}")
    assert e < 1e-3


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_config1_unipc_loop_vs_reference_golden(cuda, precision):
    """Config 1 (full base UNet, 1 prompt, CFG 3, 256 x 16) with UniPC-2 bh2 at 10 steps."""
    gd = np.load(os.path.join(GOLD, "unipc.npz"))
    cfg, embeds, mask, lat0, _ = c1.inputs()
    m = AudioDiffusion(unet_config=cfg, precision=precision).to(cuda)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=c1.SEEDS["weights"]))
    s = unipc()
    trace = []
    lat = m.inference(["synthetic prompt"], s, 10, c1.GUIDANCE, prompt_embeds=embeds, boolean_prompt_mask=mask,
                      latents=lat0, trace=trace)
    assert s.timesteps.tolist() == gd["config1_timesteps_10"].tolist()
    e = rel(lat, gd["config1_latents_10"])
    dn = max(abs(float(x.norm()) - b) / b for x, b in zip(trace, gd["config1_step_norms_10"].tolist()))
    print(f"config-1 UniPC-2 bh2 x 10 steps, {precision}: latents rel err vs REFERENCE golden {e:.3e}; worst per-step "
          f"|latents| norm deviation {dn:.3e}")
    # the bounds of the DPM-Solver config-1 loops: split 1e-3; bf16 operands through 10 CFG-amplified multistep steps
    assert e < (1e-3 if precision == "split" else 1.5e-1)
    del m
    torch.cuda.empty_cache()


def test_sharded_unipc_batch_reproduces_the_single_gpu_run(cuda, monkeypatch):
    t = Tango.from_synthetic(unet_config=synth.TINY_UNET_CONFIG, device=cuda, precision="split", scheduler="unipc")
    prompts = [f"prompt number {i}" for i in range(5)]

    def run(world, r):
        monkeypatch.setattr(parallel, "world_size", lambda: world)
        monkeypatch.setattr(parallel, "rank", lambda: r)
        monkeypatch.setattr(parallel, "allgather_waves", lambda w, dev=None: w)
        g = torch.Generator(device=cuda).manual_seed(77)
        return t.generate_for_batch(prompts, steps=5, guidance=3, batch_size=4, latent_shape=(32, 16), generator=g,
                                    shard=world > 1)

    full = run(1, 0)
    r0, r1 = run(2, 0), run(2, 1)
    assert len(full) == 5 and len(r0) == 3 and len(r1) == 2
    for got, want in zip([r0[0], r0[1], r1[0], r1[1], r0[2]], full):
        assert np.abs(got.astype(np.int32) - want.astype(np.int32)).max() <= 2


@pytest.mark.parametrize("cfg_on", [False, True])
@pytest.mark.parametrize("p,q", [(0, 1), (1, 2), (2, 2), (3, 3), (2, 1)])
def test_kernel_contract_edges(cuda, cfg_on, p, q):
    """ld_mo > C, hi/lo split_off with untouched padding columns, in-place sample and last, CFG on and off: the kernel
    equals its torch statement bit for bit (the statement's fma is exact)."""
    B, C, HW, ld_mo, so, ld_in = 2, 8, 64, 11, 10, 24
    g = torch.Generator().manual_seed(p * 10 + q)
    rnd = lambda *s: torch.randn(*s, generator=g)   # noqa: E731
    mo = rnd((2 if cfg_on else 1) * B * HW, ld_mo)
    sample, hist, last = rnd(B, C, HW), [rnd(B, C, HW) for _ in range(3)], rnd(B, C, HW)
    coef = torch.cat([torch.tensor([0.9, -0.4, 0.8]), rnd(15) * 0.3])
    coef[[6, 7, 14, 15]] = torch.tensor([-0.7, -1.6, 0.6, 1.3])
    nin = torch.full(((2 if cfg_on else 1) * B * HW, ld_in), 7.0, dtype=torch.bfloat16)
    want = {"m": torch.zeros(B, C, HW), "last": last.clone(), "prev": sample.clone(), "nin": nin.clone()}
    spec_unipc_step(mo, cfg_on, 2.5, sample, coef, p, q, want["m"], hist, want["last"], want["prev"], want["nin"], B=B,
                    Cc=C, HW=HW, split_off=so)
    d = {k: v.to(cuda) for k, v in dict(mo=mo, sample=sample, coef=coef, last=last, nin=nin).items()}
    dh = [h.to(cuda) for h in hist]
    m = torch.zeros(B, C, HW, device=cuda)
    L.unipc_step(d["mo"], cfg_on, 2.5, d["sample"], d["coef"], p, q, m, dh, d["last"], d["sample"], d["nin"], B=B,
                 Cc=C, HW=HW, split_off=so)
    torch.cuda.synchronize()
    assert torch.equal(m.cpu(), want["m"]) and torch.equal(d["sample"].cpu(), want["prev"])
    assert torch.equal(d["last"].cpu(), want["last"])
    assert torch.equal(d["nin"].cpu().view(torch.int16), want["nin"].view(torch.int16))
    assert bool((d["nin"].cpu()[:, 2 * so:].float() == 7.0).all()) and bool((d["nin"].cpu()[:, C:so].float() == 7.0).all())
