"""CPU: text-guided editing and inpainting. The scheduler arithmetic (strength -> t_start, add_noise, blend rows, the
orders of a DPM-Solver loop entered mid-grid) is held bit for bit to the fork's values in tests/golden/edit.npz
(oracle/make_golden_edit.py); the edit and inpaint loops run through cabi_spec.SPEC, whose `spec_latent_blend` is a
torch statement of tng_latent_blend. Nothing here is a CPU fallback of the product: the substitution exists only under
pytest's monkeypatch."""
import json
import os

import numpy as np
import pytest
import torch

import cabi_spec
from oracle import edit as oedit
from tango_b200 import lib as L
from tango_b200 import synth
from tango_b200.pipeline import AudioDiffusion, Tango, ratio_mask
from tango_b200.schedulers import DDIMScheduler, DDPMScheduler, DPMSolverMultistepScheduler

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CPU = torch.device("cpu")


@pytest.fixture
def spec_backend(monkeypatch):
    cabi_spec.install_spec_backend(monkeypatch)

    class _NoEvent:
        def __init__(self, *a, **k):
            pass

        def record(self, *a, **k):
            pass

        def elapsed_time(self, other):
            return 0.0

    monkeypatch.setattr(torch.cuda, "Event", _NoEvent)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)


def golden():
    gd = np.load(os.path.join(GOLD, "edit.npz"))
    return gd, json.loads(str(gd["cases"]))


SCHEDS = {"ddpm": lambda: DDPMScheduler.from_pretrained(), "ddim": lambda: DDIMScheduler.from_pretrained(),
          "dpm": lambda: DPMSolverMultistepScheduler.from_config(DDPMScheduler.from_pretrained().config)}
STRENGTHS = (0.0, 0.01, 0.1, 0.29, 0.3, 0.5, 0.6, 0.75, 0.8, 0.99, 1.0)


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


# ---------------------------------------------------------------------------------------------------- scheduler maths
def test_strength_selects_the_forks_timesteps():
    gd, _ = golden()
    assert int(100 * 0.29) == 28
    for name, make in SCHEDS.items():
        for n in (10, 25, 100):
            s = make()
            s.set_timesteps(n)
            assert s.timesteps.tolist() == gd[f"grid_{name}_{n}"].tolist()
            for st, want in zip(STRENGTHS, gd[f"t_start_{name}_{n}"].tolist()):
                if min(int(n * st), n) == 0:      # the fork fails with a shape error here; the product says why
                    with pytest.raises(ValueError, match="runs no denoising step"):
                        s.get_timesteps(n, st)
                    continue
                t_start, ts = s.get_timesteps(n, st)
                assert t_start == want == oedit.get_timesteps(n, st), (name, n, st)
                if n == 100:
                    assert ts.tolist() == gd[f"suffix_{name}_{n}_{st}"].tolist()
    s = DDPMScheduler.from_pretrained()
    s.set_timesteps(100)
    assert s.get_timesteps(100, 0.29)[0] == 72
    for bad in (-0.1, 1.01):
        with pytest.raises(ValueError, match="strength"):
            s.get_timesteps(100, bad)


def test_blend_rows_are_the_forks_add_noise_scalars():
    gd, _ = golden()
    for name, make in SCHEDS.items():
        for n in (10, 25, 100):
            s = make()
            s.set_timesteps(n)
            assert np.array_equal(s.blend_table().numpy(), gd[f"blend_{name}_{n}"]), (name, n)


def test_add_noise_bit_exact_against_the_fork(spec_backend):
    gd, _ = golden()
    x0, eps = torch.from_numpy(gd["add_noise_x0"]), torch.from_numpy(gd["add_noise_eps"])
    for name, make in SCHEDS.items():
        s = make()
        for k, t in enumerate(gd["add_noise_t"].tolist()):
            assert np.array_equal(s.add_noise(x0, eps, torch.tensor([t])).numpy(), gd[f"add_noise_{name}"][k]), (name, t)
        got = s.add_noise(x0, eps, torch.tensor([999, 500, 1]))
        assert np.array_equal(got.numpy(), gd[f"add_noise_per_sample_{name}"])
    with pytest.raises(ValueError):
        s.add_noise(x0, eps, torch.tensor([1, 2]))


def test_mid_grid_dpm_orders_match_the_fork():
    gd, _ = golden()
    rec = json.loads(str(gd["dpm_orders"]))
    assert len(rec) == 30
    for key, want in rec.items():
        order, n, st = key.split("_")
        s = SCHEDS["dpm"]()
        s = DPMSolverMultistepScheduler.from_config(s.config, solver_order=int(order))
        s.set_timesteps(int(n))
        t_start = oedit.get_timesteps(int(n), float(st))
        tab = s.loop_table(CPU, t_start)
        assert s._loop_orders[t_start:] == want, key
        for i in range(t_start, int(n)):
            assert torch.equal(tab[i], s._coefficients_at(i, want[i - t_start]))
    s = SCHEDS["dpm"]()
    s.set_timesteps(25)
    full = s.coefficient_table().clone()
    s.loop_table(CPU, 10)
    assert torch.equal(s.loop_table(CPU, 0), full) and torch.equal(s.coefficient_table(), full)
    assert s._loop_orders == s._orders


def test_ratio_masks_follow_audioldm():
    gd, cases = golden()
    for H, W, tb, fb in ((32, 16, (0.25, 0.5), (0.5, 0.75)), (256, 16, (0.1, 0.37), None), (256, 16, None, (0.0, 0.3)),
                         (256, 16, (1.0, 1.0), (1.0, 1.0))):
        m = ratio_mask(H, W, tb, fb)
        assert m.shape == (1, 1, H, W) and torch.equal(m, oedit.ratio_mask(H, W, tb, fb))
        # ldm.py:773-777, written out
        ref = torch.ones(1, H, W)
        if tb is not None:
            ref[:, int(H * tb[0]):int(H * tb[1]), :] = 0
        if fb is not None:
            ref[:, :, int(W * fb[0]):int(W * fb[1])] = 0
        assert torch.equal(m[:, 0], ref)
    c = cases["tiny_ddim_inpaint"]
    assert np.array_equal(ratio_mask(32, 16, c["time_band"], c["freq_band"]).numpy(), gd["tiny_ddim_inpaint_mask"])
    assert bool((ratio_mask(8, 4, (1.0, 1.0), (1.0, 1.0)) == 1).all())


# ---------------------------------------------------------------------------------------------------- the loop
def tiny_model(precision="split"):
    cfg = synth.TINY_UNET_CONFIG
    m = AudioDiffusion(unet_config=cfg, precision=precision, use_cuda_graph=False).to(CPU)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    return m


def case_kwargs(gd, cases, name):
    """The edit inputs of golden case `name`: its clip's x0 (stored) and the fork's draws (regenerated from the seed)."""
    c = cases[name]
    H = c["latent_shape"][0]
    _, noise, step_noises = oedit.seeded_draws(c["seed"], (1, 8, H, 16), c["step_draws"])
    kw = dict(init_latents=torch.from_numpy(gd[c["x0_key"]]), init_noise=noise, noises=step_noises, latent_shape=(H, 16))
    if name + "_mask" in gd:
        kw["inpaint_mask"] = torch.from_numpy(gd[name + "_mask"])
    return kw


@pytest.mark.parametrize("name", ["tiny_ddpm", "tiny_ddim_inpaint", "tiny_dpm"])
def test_tiny_edit_loops_match_the_fork_pipelines(spec_backend, name):
    gd, cases = golden()
    c = cases[name]
    m = tiny_model()
    sch = SCHEDS[c["scheduler"]]()
    blends = []
    orig = L.latent_blend
    L.latent_blend = lambda *a, **k: (blends.append(a[2] is not None), orig(*a, **k))[1]
    try:
        trace = []
        ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
        lat = m.inference(["synthetic prompt"], sch, c["steps"], c["guidance"], strength=c["strength"], trace=trace,
                          prompt_embeds=torch.from_numpy(ti["embeds"]), boolean_prompt_mask=torch.from_numpy(ti["mask"]),
                          **case_kwargs(gd, cases, name))
    finally:
        L.latent_blend = orig
    n_run = c["steps"] - c["t_start"]
    assert len(trace) == n_run
    masked = c["time_band"] is not None or c["freq_band"] is not None
    assert blends == [False] + ([True] * (n_run + 1) if masked else [])
    if c["scheduler"] == "dpm":
        assert sch._loop_orders[c["t_start"]:] == c["orders"]
    e = rel(lat, gd[name + "_latents"])
    assert e < 1e-3, e
    if masked:   # kept positions are the input latents exactly
        keep = torch.from_numpy(gd[name + "_mask"]).expand_as(lat) == 1
        assert torch.equal(lat[keep], torch.from_numpy(gd[c["x0_key"]])[keep])


def test_default_path_is_unchanged_without_edit_keywords(spec_backend):
    """No edit keyword: no blend launch, same latents as the plain loop (the generation path)."""
    ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    m = tiny_model()
    calls = []
    orig = L.latent_blend
    L.latent_blend = lambda *a, **k: (calls.append(1), orig(*a, **k))[1]
    try:
        lat = m.inference(["p"], DDPMScheduler.from_pretrained(), 4, 3.0, prompt_embeds=torch.from_numpy(ti["embeds"]),
                          boolean_prompt_mask=torch.from_numpy(ti["mask"]), latents=torch.from_numpy(ti["lat0"]),
                          noises=list(torch.from_numpy(ti["noises"])), latent_shape=(32, 16))
    finally:
        L.latent_blend = orig
    assert calls == [] and rel(lat, ti["latents"]) < 1e-3


def test_refusals(spec_backend):
    m = tiny_model()
    ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    kw = dict(prompt_embeds=torch.from_numpy(ti["embeds"]), boolean_prompt_mask=torch.from_numpy(ti["mask"]),
              latent_shape=(32, 16))
    x0 = torch.zeros(1, 8, 32, 16)
    for bad in (dict(init_latents=x0, strength=1.5), dict(init_latents=x0, strength=-0.5),
                dict(init_latents=x0, strength=0.05), dict(init_noise=x0), dict(strength=0.5),
                dict(init_latents=x0, latents=x0), dict(init_latents=torch.zeros(1, 8, 16, 16)),
                dict(init_latents=x0, inpaint_mask=torch.full((1, 1, 32, 16), 2.0)),
                dict(init_latents=x0, inpaint_mask=torch.ones(1, 32, 16))):
        with pytest.raises(ValueError):
            m.inference(["p"], DDPMScheduler.from_pretrained(), 10, 3.0, **kw, **bad)


# ---------------------------------------------------------------------------------------------------- façade + RNG
def synthetic_tango():
    t = Tango.from_synthetic(unet_config=synth.TINY_UNET_CONFIG, device="cpu", precision="split")
    t.model.use_cuda_graph = False
    return t


def test_synthetic_encoder_weights_leave_the_decoder_unchanged():
    both = synth.synth_state_dict(dict(synth.vae_decoder_param_shapes(), **synth.vae_encoder_param_shapes()), seed=0)
    dec = synth.synth_state_dict(synth.vae_decoder_param_shapes(), seed=0)
    assert all(torch.equal(both[k], v) for k, v in dec.items())
    assert synthetic_tango().vae.has_encoder


def test_edit_needs_cuda_and_an_encoder():
    t = synthetic_tango()
    wave = np.zeros(32 * 4 * 160, dtype=np.int16)
    with pytest.raises(L.TangoB200Error):
        t.edit("rain", wave, strength=0.5, steps=4, latent_shape=(32, 16))
    t.vae.load_state_dict(synth.synth_state_dict(synth.vae_decoder_param_shapes(), seed=0))
    with pytest.raises(L.TangoB200Error, match="encoder"):
        t.edit("rain", wave, strength=0.5, steps=4, latent_shape=(32, 16))


def test_rng_draw_order_and_empty_shard_accounting(spec_backend, monkeypatch):
    """Draws: the posterior noise of the clips, the add-noise draw of the batch, one DDPM draw per executed step with
    t > 0; advance_rng consumes exactly the same stream."""
    t = synthetic_tango()
    shapes = []
    orig = AudioDiffusion.randn_rows
    monkeypatch.setattr(AudioDiffusion, "randn_rows",
                        staticmethod(lambda shape, *a, **k: (shapes.append(tuple(shape)), orig(shape, *a, **k))[1]))
    monkeypatch.setattr(Tango, "_decode", lambda self, lat: np.zeros((lat.shape[0], 4), dtype=np.int16))
    g = torch.Generator().manual_seed(3)
    clips = [np.sin(np.arange(32 * 4 * 160) * f).astype(np.float32) for f in (0.01, 0.02)]
    waves = t.edit_for_batch(["rain", "thunder"], clips, strength=0.5, steps=4, guidance=3, latent_shape=(32, 16),
                             generator=g)
    assert len(waves) == 2
    # DDPM 4-step grid [750, 500, 250, 0]; strength 0.5 runs [250, 0]: one step draws
    assert shapes == [(2, 8, 32, 16), (2, 8, 32, 16), (2, 8, 32, 16)]
    g2 = torch.Generator().manual_seed(3)
    t.model.advance_rng(2, t.scheduler, 4, g2, (32, 16), edit_clips=2, strength=0.5)
    assert torch.equal(torch.randn(5, generator=g), torch.randn(5, generator=g2))
    # one clip serving both prompts draws one posterior row
    shapes.clear()
    t.edit_for_batch(["rain", "thunder"], clips[0], strength=0.5, steps=4, guidance=3, latent_shape=(32, 16),
                     generator=torch.Generator().manual_seed(3))
    assert shapes[0] == (1, 8, 32, 16) and shapes[1] == (2, 8, 32, 16)
