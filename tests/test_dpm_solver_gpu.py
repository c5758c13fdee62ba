"""GPU: the multistep DPM-Solver(++) scheduler on tng_dpm_step, against the fork's scheduler run through the unmodified
reference (tests/golden/dpm_solver.npz, oracle/make_golden_dpm.py): `step` bit for bit over the whole supported matrix,
the tiny CFG loop, config 1 at full size at 10 and 25 steps, and the prompt-sharded batch path."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_config1 as c1
from tango_b200 import parallel, synth
from tango_b200.pipeline import AudioDiffusion, Tango
from tango_b200.schedulers import DDPMScheduler, DPMSolverMultistepScheduler

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def dpm(**kw):
    return DPMSolverMultistepScheduler.from_config(DDPMScheduler.from_pretrained().config, **kw)


def test_step_bit_exact_over_every_golden_loop(cuda):
    gd = np.load(os.path.join(GOLD, "dpm_solver.npz"))
    mat = json.loads(str(gd["loop_configs"]))
    n = 4 * 3 * 8 * 8
    x_fork = (torch.arange(n).reshape(3, 8, 8, 4) / n).permute(3, 0, 1, 2).contiguous()
    for k, (kw, steps, model) in enumerate(mat):
        s = DPMSolverMultistepScheduler(**kw)
        s.set_timesteps(steps, device=cuda)
        x = (torch.from_numpy(gd["sin_x0"]) if model == "sin" else x_fork).to(cuda)
        for t in s.timesteps:
            xc, tc = x.cpu(), t.cpu()     # the model is evaluated on the CPU, as in the golden generator
            mo = torch.sin(xc * 3.0 + float(tc) / 1000) if model == "sin" else xc * tc / (tc + 1)
            x = s.step(mo.to(cuda), t, x).prev_sample
        assert np.array_equal(x.cpu().numpy(), gd[f"loop_{k}"]), f"loop {k} {kw} {steps} steps not bit-exact"


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_tiny_inference_vs_golden(cuda, precision):
    gd, ti = np.load(os.path.join(GOLD, "dpm_solver.npz")), np.load(os.path.join(GOLD, "tiny_inference.npz"))
    cfg = synth.TINY_UNET_CONFIG
    sd = synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0)
    kw = dict(prompt_embeds=torch.from_numpy(ti["embeds"]), boolean_prompt_mask=torch.from_numpy(ti["mask"]),
              latents=torch.from_numpy(ti["lat0"]), latent_shape=(32, 16))
    m = AudioDiffusion(unet_config=cfg, precision=precision).to(cuda)
    m.unet.load_state_dict(sd)
    lat = m.inference(["synthetic prompt"], dpm(), 6, 3.0, **kw).clone()
    e = rel(lat, gd["tiny_latents"])
    print(f"tiny 6-step DPM-Solver++ 2M CFG loop {precision}: rel err vs reference golden {e:.3e}")
    assert e < (1e-3 if precision == "split" else 6e-2)
    # a second call on the same shape reuses the graph and the history slots: same result
    again = m.inference(["synthetic prompt"], dpm(), 6, 3.0, **kw)
    assert rel(again, lat) < (1e-4 if precision == "split" else 6e-2)
    m2 = AudioDiffusion(unet_config=cfg, precision=precision, use_cuda_graph=False).to(cuda)
    m2.unet.load_state_dict(sd)
    lat2 = m2.inference(["synthetic prompt"], dpm(), 6, 3.0, **kw)
    # GroupNorm statistics are reduced with atomics: graph replay and eager agree to round-off (bounds as for DDPM)
    assert rel(lat, lat2) < (1e-4 if precision == "split" else 6e-2)


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_config1_dpm_loop_vs_reference_golden(cuda, precision):
    """Config 1 (full base UNet, 1 prompt, CFG 3, 256 x 16) with DPM-Solver++ 2M at 10 and 25 steps."""
    gd = np.load(os.path.join(GOLD, "dpm_solver.npz"))
    cfg, embeds, mask, lat0, _ = c1.inputs()
    m = AudioDiffusion(unet_config=cfg, precision=precision).to(cuda)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=c1.SEEDS["weights"]))
    for steps in (10, 25):
        s = dpm()
        trace = []
        lat = m.inference(["synthetic prompt"], s, steps, c1.GUIDANCE, prompt_embeds=embeds, boolean_prompt_mask=mask,
                          latents=lat0, trace=trace)
        assert s.timesteps.tolist() == gd[f"config1_timesteps_{steps}"].tolist()
        e = rel(lat, gd[f"config1_latents_{steps}"])
        norms = [float(x.norm()) for x in trace]
        dn = max(abs(a - b) / b for a, b in zip(norms, gd[f"config1_step_norms_{steps}"].tolist()))
        print(f"config-1 DPM-Solver++ 2M x {steps} steps, {precision}: latents rel err vs REFERENCE golden {e:.3e}; "
              f"worst per-step |latents| norm deviation {dn:.3e}")
        if precision == "split":
            assert e < 1e-3
        else:
            # bf16 operands, ~1e-2 per forward, through 10-25 CFG-amplified steps of a second-order multistep
            # solver; stated bound 1.5e-1 (as for the DDPM / DDIM config-1 loops), measured value printed above
            assert e < 1.5e-1
    del m
    torch.cuda.empty_cache()


def test_sharded_dpm_batch_reproduces_the_single_gpu_run(cuda, monkeypatch):
    """Ranks 0 and 1 of a world of 2, run one after the other on one device with the same seed, give the one-GPU
    waveforms: the DPM-Solver draws only the initial latents, so an empty shard's rank has nothing else to skip."""
    t = Tango.from_synthetic(unet_config=synth.TINY_UNET_CONFIG, device=cuda, precision="split")
    t.scheduler = DPMSolverMultistepScheduler.from_config(t.scheduler.config)
    prompts = [f"prompt number {i}" for i in range(5)]           # chunks of 4 + 1: the second chunk leaves rank 1 empty

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
