"""GPU: text-guided editing and inpainting on tng_latent_blend, against the fork's img2img / legacy-inpaint pipelines
run through the unmodified reference (tests/golden/edit.npz, oracle/make_golden_edit.py)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import edit as oedit
from oracle import make_golden_config1 as c1
from tango_b200 import lib as L
from tango_b200 import parallel, synth
from tango_b200.pipeline import AudioDiffusion, Tango
from tango_b200.schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler
from cabi_spec import spec_latent_blend
from test_edit_cpu import case_kwargs

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
SCHEDS = {"ddpm": lambda: DDPMScheduler.from_pretrained(), "ddim": lambda: DDIMScheduler.from_pretrained(),
          "dpm": lambda: DPMSolverMultistepScheduler.from_config(DDPMScheduler.from_pretrained().config)}


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def golden():
    gd = np.load(os.path.join(GOLD, "edit.npz"))
    return gd, json.loads(str(gd["cases"]))


@pytest.mark.parametrize("B,Cc,H,W", [(2, 8, 32, 16), (3, 8, 7, 13), (1, 4, 5, 3)])
def test_latent_blend_bit_exact_against_its_statement(cuda, B, Cc, H, W):
    """No mask, one broadcast mask and per-sample masks; CFG on and off; bf16 and hi/lo packing; ragged B*H*W."""
    g = torch.Generator().manual_seed(B * 100 + H)
    HW = H * W
    x0, nz, s0 = (torch.randn(B, Cc, H, W, generator=g) for _ in range(3))
    coef = torch.tensor([0.83, 0.557])
    masks = [None, torch.rand(1, HW, generator=g), (torch.rand(B, HW, generator=g) > 0.5).float()]
    for mask in masks:
        for noise in (nz, None):
            for cfg in (False, True):
                for split_off in (0, Cc):
                    ld = Cc + split_off + 3
                    rows = (2 if cfg else 1) * B * HW
                    want_s = s0.clone()
                    want_in = torch.full((rows, ld), float("nan"), dtype=torch.bfloat16)
                    spec_latent_blend(x0, noise, mask, coef, want_s, want_in, B=B, Cc=Cc, HW=HW, cfg=cfg,
                                      split_off=split_off)
                    got_s = s0.clone().to(cuda)
                    got_in = torch.full((rows, ld), float("nan"), dtype=torch.bfloat16, device=cuda)
                    L.latent_blend(x0.to(cuda), None if noise is None else noise.to(cuda),
                                   None if mask is None else mask.to(cuda), coef.to(cuda), got_s, got_in, B=B, Cc=Cc,
                                   HW=HW, cfg=cfg, split_off=split_off)
                    torch.cuda.synchronize()
                    assert torch.equal(got_s.cpu(), want_s), (mask is None, noise is None, cfg, split_off)
                    gi, wi = got_in.cpu().float(), want_in.float()
                    assert torch.equal(gi.isnan(), wi.isnan())      # the padding columns stay untouched
                    assert torch.equal(gi.nan_to_num(), wi.nan_to_num())


def test_add_noise_bit_exact_against_the_fork(cuda):
    gd, _ = golden()
    x0, eps = torch.from_numpy(gd["add_noise_x0"]).to(cuda), torch.from_numpy(gd["add_noise_eps"]).to(cuda)
    for name, make in SCHEDS.items():
        s = make()
        for k, t in enumerate(gd["add_noise_t"].tolist()):
            assert np.array_equal(s.add_noise(x0, eps, torch.tensor([t])).cpu().numpy(), gd[f"add_noise_{name}"][k])
        got = s.add_noise(x0, eps, torch.tensor([999, 500, 1]))
        assert np.array_equal(got.cpu().numpy(), gd[f"add_noise_per_sample_{name}"])


def check_kept_positions(lat, gd, cases, name):
    """With a binary mask every kept position holds x0 bit for bit."""
    if name + "_mask" not in gd:
        return
    keep = torch.from_numpy(gd[name + "_mask"]).to(lat.device).expand_as(lat) == 1
    assert torch.equal(lat[keep], torch.from_numpy(gd[cases[name]["x0_key"]]).to(lat.device)[keep])


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_tiny_edit_loops_vs_golden(cuda, precision):
    gd, cases = golden()
    ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    cfg = synth.TINY_UNET_CONFIG
    m = AudioDiffusion(unet_config=cfg, precision=precision).to(cuda)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    cond = dict(prompt_embeds=torch.from_numpy(ti["embeds"]), boolean_prompt_mask=torch.from_numpy(ti["mask"]))
    for name in ("tiny_ddpm", "tiny_ddim_inpaint", "tiny_dpm"):
        c = cases[name]
        kw = dict(cond, strength=c["strength"], **case_kwargs(gd, cases, name))
        lat = m.inference(["synthetic prompt"], SCHEDS[c["scheduler"]](), c["steps"], c["guidance"], **kw).clone()
        e = rel(lat, gd[name + "_latents"])
        print(f"tiny {name} ({c['scheduler']}, strength {c['strength']}) {precision}: rel err vs reference golden {e:.3e}")
        # split: fp32-faithful operands; bf16: ~1e-2 per forward through <= 8 CFG steps (as the DPM tiny bound)
        assert e < (1e-3 if precision == "split" else 6e-2)
        check_kept_positions(lat, gd, cases, name)
        graphs = len(m._state)
        again = m.inference(["synthetic prompt"], SCHEDS[c["scheduler"]](), c["steps"], c["guidance"], **kw)
        assert len(m._state) == graphs            # same shape: the captured UNet graph is reused
        assert rel(again, lat) < (1e-4 if precision == "split" else 6e-2)
        check_kept_positions(again, gd, cases, name)


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_config1_edit_and_inpaint_vs_golden(cuda, precision):
    gd, cases = golden()
    cfg, embeds, mask, _, _ = c1.inputs()
    m = AudioDiffusion(unet_config=cfg, precision=precision).to(cuda)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=c1.SEEDS["weights"]))
    for name in ("config1_edit", "config1_inpaint"):
        c = cases[name]
        lat = m.inference(["synthetic prompt"], SCHEDS[c["scheduler"]](), c["steps"], c["guidance"],
                          prompt_embeds=embeds, boolean_prompt_mask=mask, strength=c["strength"],
                          **case_kwargs(gd, cases, name))
        e = rel(lat, gd[name + "_latents"])
        print(f"config-1 {name} ({c['scheduler']}, strength {c['strength']}) {precision}: latents rel err vs reference "
              f"golden {e:.3e}")
        # bf16: the config-1 bound of the DDPM / DDIM / DPM loops; measured value printed above
        assert e < (1e-3 if precision == "split" else 1.5e-1)
        check_kept_positions(lat, gd, cases, name)
    del m
    torch.cuda.empty_cache()


def test_tango_edit_end_to_end(cuda):
    """Waveform -> STFT -> VAE encoder -> edit loop -> decode, with a CPU generator seeded like the golden: the draws
    are the fork's, so the latents follow the reference up to the front end's and the UNet's kernel round-off."""
    gd, cases = golden()
    c = cases["tiny_ddpm"]
    t = Tango.from_synthetic(unet_config=synth.TINY_UNET_CONFIG, device=cuda, precision="split")
    ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    got = {}
    orig = t._decode
    t._decode = lambda lat: (got.setdefault("lat", lat.clone()), orig(lat))[1]
    clip = oedit.input_wave(4 * 32 * synth.STFT_CONFIG["hop_length"], c["seed"])
    wave = t.edit("synthetic prompt", clip, strength=c["strength"], steps=c["steps"],
                  guidance=c["guidance"], latent_shape=(32, 16), generator=torch.Generator().manual_seed(c["seed"]),
                  prompt_embeds=torch.from_numpy(ti["embeds"]), boolean_prompt_mask=torch.from_numpy(ti["mask"]))
    assert wave.dtype == np.int16 and wave.shape == gd["tiny_ddpm_decoded_wave_i16"].shape[1:]
    e = rel(got["lat"], gd["tiny_ddpm_latents"])
    print(f"Tango.edit end to end (split): latents rel err vs reference golden {e:.3e}")
    assert e < 1e-2
    inp = t.edit("synthetic prompt", clip, strength=0.5, steps=10, latent_shape=(32, 16),
                 time_mask_ratio_start_and_end=(0.25, 0.75), generator=torch.Generator().manual_seed(1),
                 prompt_embeds=torch.from_numpy(ti["embeds"]), boolean_prompt_mask=torch.from_numpy(ti["mask"]))
    assert inp.dtype == np.int16 and inp.shape == wave.shape


def test_sharded_edit_batch_reproduces_the_single_gpu_run(cuda, monkeypatch):
    """Ranks 0 and 1 of a world of 2, run one after the other on one device with the same seed, give the one-GPU
    waveforms; DDPM draws per step, so the empty-shard rank must skip the posterior, add-noise and step draws."""
    t = Tango.from_synthetic(unet_config=synth.TINY_UNET_CONFIG, device=cuda, precision="split")
    prompts = [f"prompt number {i}" for i in range(5)]           # chunks of 4 + 1: the second chunk leaves rank 1 empty
    g0 = torch.Generator().manual_seed(9)
    clips = [torch.randn(32 * 4 * 160, generator=g0) * 0.3 for _ in prompts]

    def run(world, r):
        monkeypatch.setattr(parallel, "world_size", lambda: world)
        monkeypatch.setattr(parallel, "rank", lambda: r)
        monkeypatch.setattr(parallel, "allgather_waves", lambda w, dev=None: w)
        g = torch.Generator(device=cuda).manual_seed(77)
        return t.edit_for_batch(prompts, clips, strength=0.6, steps=5, guidance=3, batch_size=4, latent_shape=(32, 16),
                                generator=g, shard=world > 1, time_mask_ratio_start_and_end=(0.5, 1.0))

    full = run(1, 0)
    r0, r1 = run(2, 0), run(2, 1)
    assert len(full) == 5 and len(r0) == 3 and len(r1) == 2
    for got, want in zip([r0[0], r0[1], r1[0], r1[1], r0[2]], full):
        assert np.abs(got.astype(np.int32) - want.astype(np.int32)).max() <= 2
