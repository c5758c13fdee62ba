"""Pin oracle/edit.py against the UNMODIFIED fork img2img / legacy-inpaint pipelines and write tests/golden/edit.npz,
with what each part measured in tests/golden/edit.json (TEST INFRASTRUCTURE ONLY; build container only, ~10 min on 8
cores).

    python -m oracle.make_golden_edit

The fork's `StableDiffusionImg2ImgPipeline.__call__` and `StableDiffusionInpaintPipelineLegacy.__call__` run unbound
on a stand-in `self` that supplies the oracle UNet (with the attention mask bound), the fork's scheduler, a VAE whose
`encode` wraps the reference AudioLDM encoder's moments in the fork's DiagonalGaussianDistribution and whose
`decode_latents` returns the latents, a pass-through safety checker and the prompt embeddings. The generator is a
seeded CPU torch.Generator, so the fork's own draw order (posterior, add-noise, DDPM steps) is what is recorded; the
oracle replays the recorded draws. Stored:
  * strength -> t_start / executed timesteps for DDPM, DDIM and DPM-Solver over a strength grid (fork get_timesteps);
  * the fork's add_noise values and its alphas_cumprod ** 0.5 / (1 - alphas_cumprod) ** 0.5 per grid;
  * the update order of every executed DPM-Solver step of loops entered mid-grid;
  * per latent size: the clean latents x0 of the shared input clip (for the tiny clip also its mel and the encoder's
    moments); per case: final latents, per-step latent norms and the mask; for one tiny case also the reference decode
    (mel, int16 waveform). The input clips and the random draws follow from the seeds and are asserted, not stored.
"""
from __future__ import annotations

import contextlib
import json
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import dpm_solver as odpm  # noqa: E402
from oracle import edit as oedit  # noqa: E402
from oracle import make_golden_config1 as mg1  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle import schedulers as osched  # noqa: E402
from oracle import stft as ostft  # noqa: E402
from oracle import unet as ounet  # noqa: E402
from tango_b200 import stft as pstft  # noqa: E402
from tango_b200 import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SC = dict(osched.SD21_CONFIG)
STRENGTHS = (0.0, 0.01, 0.1, 0.29, 0.3, 0.5, 0.6, 0.75, 0.8, 0.99, 1.0)
GRID_STEPS = (10, 25, 100)
# name: (unet, H, scheduler, steps, strength, time band, freq band, guidance, seed)
CASES = {
    "tiny_ddpm": ("tiny", 32, "ddpm", 10, 0.6, None, None, 3.0, 11),
    "tiny_ddim_inpaint": ("tiny", 32, "ddim", 10, 0.8, (0.25, 0.5), (0.5, 0.75), 3.0, 11),
    "tiny_dpm": ("tiny", 32, "dpm", 10, 0.5, None, None, 3.0, 11),
    "config1_edit": ("base", 256, "ddim", 10, 0.6, None, None, mg1.GUIDANCE, 21),
    "config1_inpaint": ("base", 256, "ddpm", 10, 0.5, (0.5, 0.75), None, mg1.GUIDANCE, 21),
}
# The cases of one latent size edit the same seeded clip with the same seed, so they share one x0; the clip and every
# random draw are regenerated from the seed (oracle/edit.py: input_wave, seeded_draws) and are not stored.
DECODED = "tiny_ddpm"


def import_pipelines():
    """Import the two fork pipeline modules unmodified through refshim."""
    refshim.install()
    import transformers.utils as tu
    if not hasattr(tu, "FLAX_WEIGHTS_NAME"):
        tu.FLAX_WEIGHTS_NAME = "flax_model.msgpack"
    base = os.path.join(refshim.DIFFUSERS_SRC, "pipelines")
    refshim._pkg("diffusers.pipelines", base)
    sd_pkg = refshim._pkg("diffusers.pipelines.stable_diffusion", os.path.join(base, "stable_diffusion"))

    class StableDiffusionPipelineOutput(types.SimpleNamespace):
        pass

    sd_pkg.StableDiffusionPipelineOutput = StableDiffusionPipelineOutput
    sd_pkg.StableDiffusionSafetyChecker = type("StableDiffusionSafetyChecker", (), {})
    import importlib
    i2i = importlib.import_module("diffusers.pipelines.stable_diffusion.pipeline_stable_diffusion_img2img")
    inp = importlib.import_module("diffusers.pipelines.stable_diffusion.pipeline_stable_diffusion_inpaint_legacy")
    return i2i.StableDiffusionImg2ImgPipeline, inp.StableDiffusionInpaintPipelineLegacy


def fork_schedulers():
    from diffusers.schedulers.scheduling_ddim import DDIMScheduler
    from diffusers.schedulers.scheduling_ddpm import DDPMScheduler
    DPM = odpm.reference_class()
    common = dict(num_train_timesteps=1000, beta_start=SC["beta_start"], beta_end=SC["beta_end"],
                  beta_schedule=SC["beta_schedule"], prediction_type=SC["prediction_type"])
    return {"ddpm": lambda **kw: DDPMScheduler(**common, clip_sample=False),
            "ddim": lambda **kw: DDIMScheduler(**common, clip_sample=False, set_alpha_to_one=False, steps_offset=1),
            "dpm": lambda **kw: DPM(**common, **kw)}


def oracle_scheduler(name):
    return {"ddpm": lambda: osched.OracleDDPM(**SC), "ddim": lambda: osched.OracleDDIM(**SC),
            "dpm": lambda: odpm.OracleDPMSolverMultistep(**SC)}[name]()


def record_dpm_orders(sched):
    """Wrap the fork scheduler's update methods so that each `step` appends the order it took."""
    orders = []
    for k, name in ((1, "dpm_solver_first_order_update"), (2, "multistep_dpm_solver_second_order_update"),
                    (3, "multistep_dpm_solver_third_order_update")):
        fn = getattr(sched, name)
        setattr(sched, name, (lambda f, k: lambda *a, **kw: (orders.append(k), f(*a, **kw))[1])(fn, k))
    return orders


class _Progress:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def update(self):
        pass


def stand_in(cls, unet_sd, unet_cfg, mask, scheduler, ref_vae, record):
    """The `self` of the fork pipeline `__call__`s (see the module docstring). `record` collects the moments."""
    from diffusers.models.vae import DiagonalGaussianDistribution as ForkDGD
    s = types.SimpleNamespace()
    for name in ("check_inputs", "get_timesteps", "prepare_latents", "prepare_extra_step_kwargs", "_encode_prompt"):
        setattr(s, name, types.MethodType(getattr(cls, name), s))

    def unet(x, t, encoder_hidden_states=None, **_):
        return types.SimpleNamespace(sample=ounet.unet_forward(unet_sd, unet_cfg, x, t, encoder_hidden_states, mask))

    def encode(image):
        moments = ref_vae.encode(image).parameters
        record["moments"] = moments.clone()
        return types.SimpleNamespace(latent_dist=ForkDGD(moments))

    s.unet = unet
    s.scheduler = scheduler
    s.vae = types.SimpleNamespace(encode=encode, config=types.SimpleNamespace(scaling_factor=ref_vae.scale_factor))
    s.vae_scale_factor = 1                     # the mask is given at latent resolution
    s.decode_latents = lambda latents: latents
    s.safety_checker = None
    s.run_safety_checker = lambda image, device, dtype: (image, None)
    s.image_processor = types.SimpleNamespace(preprocess=lambda image: image)
    s.text_encoder = types.SimpleNamespace(dtype=torch.float32)
    s._execution_device = s.device = torch.device("cpu")
    s.progress_bar = lambda total=None: _Progress()
    return s


class RecordingGenerator:
    """Records every tensor drawn through the fork's randn_tensor (in draw order) from one seeded CPU generator."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)
        self.draws = []


@contextlib.contextmanager
def recording(rec):
    import diffusers.models.vae as fvae
    import diffusers.schedulers.scheduling_ddpm as fddpm
    import diffusers.pipelines.stable_diffusion.pipeline_stable_diffusion_img2img as fi2i
    import diffusers.pipelines.stable_diffusion.pipeline_stable_diffusion_inpaint_legacy as finp
    from diffusers.utils import torch_utils
    orig = torch_utils.randn_tensor

    def randn(shape, generator=None, device=None, dtype=None, layout=None):
        t = orig(shape, generator=generator, device=device, dtype=dtype, layout=layout)
        rec.draws.append(t.clone())
        return t

    mods = [m for m in (fvae, fddpm, fi2i, finp) if hasattr(m, "randn_tensor")]
    for m in mods:
        m.randn_tensor = randn
    try:
        yield
    finally:
        for m in mods:
            m.randn_tensor = orig


def front_end(wave, frames):
    """wav_to_fbank at the product's STFT config (1024 / 160 / 1024, 64 slaney mel bins, 0-8 kHz) on oracle/stft.py
    (pinned to the reference torch_tools / TacotronSTFT by make_golden_stft) -> mel (1, 1, frames, 64)."""
    c = synth.STFT_CONFIG
    basis = ostft.forward_basis(c["filter_length"], c["win_length"])
    mel_basis = pstft.slaney_mel_basis(c["sampling_rate"], c["filter_length"], c["n_mel_channels"], c["mel_fmin"],
                                       c["mel_fmax"])
    fb, _, _ = ostft.wav_to_fbank([wave], basis, mel_basis, target_length=frames, filter_length=c["filter_length"],
                                  hop_length=c["hop_length"])
    return fb.unsqueeze(1).contiguous()


def maxdiff(a, b):
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max())


def scheduler_part(out, checks, scheds, I2I):
    """Strength grid, add_noise / blend rows and mid-grid DPM orders, all from the fork's own objects."""
    for name, make in scheds.items():
        for n in GRID_STEPS:
            s = make()
            s.set_timesteps(n)
            stub = types.SimpleNamespace(scheduler=s)
            out[f"grid_{name}_{n}"] = s.timesteps.numpy()
            tstarts = []
            for st in STRENGTHS:
                ts, nrun = I2I.get_timesteps(stub, n, st, "cpu")
                tstarts.append(n - nrun)
                assert oedit.get_timesteps(n, st) == n - nrun
                if n == 100:
                    out[f"suffix_{name}_{n}_{st}"] = ts.numpy()
            out[f"t_start_{name}_{n}"] = np.asarray(tstarts, dtype=np.int64)
            ac = s.alphas_cumprod[s.timesteps]
            out[f"blend_{name}_{n}"] = torch.stack([ac ** 0.5, (1 - ac) ** 0.5], 1).numpy()
    g = torch.Generator().manual_seed(5)
    x0, eps = torch.randn(3, 8, 4, 4, generator=g), torch.randn(3, 8, 4, 4, generator=g)
    out["add_noise_x0"], out["add_noise_eps"] = x0.numpy(), eps.numpy()
    ts = [999, 901, 500, 41, 1, 0]
    out["add_noise_t"] = np.asarray(ts, dtype=np.int64)
    worst = 0.0
    for name, make in scheds.items():
        s = make()
        vals = torch.stack([s.add_noise(x0, eps, torch.tensor([t])) for t in ts])
        out[f"add_noise_{name}"] = vals.numpy()
        per = s.add_noise(x0, eps, torch.tensor([999, 500, 1]))           # one timestep per sample
        out[f"add_noise_per_sample_{name}"] = per.numpy()
        orc = torch.stack([oedit.add_noise(s.alphas_cumprod, x0, eps, t) for t in ts])
        worst = max(worst, maxdiff(vals, orc))
    assert worst == 0.0, worst
    checks["add_noise_oracle_vs_fork_max_abs"] = worst
    # DPM-Solver loops entered mid-grid: the fork counts lower_order_nums from the first executed step
    orders = {}
    for order in (2, 3):
        for n in (10, 15, 25):
            for st in (0.3, 0.5, 0.6, 0.8, 1.0):
                s = scheds["dpm"](solver_order=order)
                s.set_timesteps(n)
                rec = record_dpm_orders(s)
                t_start = oedit.get_timesteps(n, st)
                x = torch.zeros(1, 1, 2, 2)
                for t in s.timesteps[t_start:]:
                    x = s.step(torch.zeros_like(x), t, x).prev_sample
                orders[f"{order}_{n}_{st}"] = rec
    out["dpm_orders"] = np.asarray(json.dumps(orders))


def main():
    torch.set_grad_enabled(False)
    t00 = time.time()
    I2I, INP = import_pipelines()
    scheds = fork_schedulers()
    out, checks = {}, {}
    scheduler_part(out, checks, scheds, I2I)
    print(f"scheduler arithmetic: fork == oracle bit for bit ({time.time() - t00:.0f} s)", flush=True)

    A = refshim.autoencoder_class()
    ref_vae = A(**synth.VAE_CONFIG).eval()
    vsd = synth.synth_state_dict(dict(synth.vae_decoder_param_shapes(), **synth.vae_encoder_param_shapes()), seed=0)
    full = ref_vae.state_dict()
    full.update(vsd)
    ref_vae.load_state_dict(full, strict=True)
    ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    cases = {}
    only = sys.argv[1:]
    for name, (unet, H, sname, steps, strength, tband, fband, guidance, seed) in CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        if unet == "tiny":
            ucfg = dict(synth.TINY_UNET_CONFIG)
            usd = synth.synth_state_dict(synth.unet_param_shapes(ucfg), seed=0)
            embeds, mask = torch.from_numpy(ti["embeds"]), torch.from_numpy(ti["mask"])
        else:
            ucfg, embeds, mask, _, _ = mg1.inputs()
            usd = synth.synth_state_dict(synth.unet_param_shapes(ucfg), seed=mg1.SEEDS["weights"])
        wave = oedit.input_wave(4 * H * synth.STFT_CONFIG["hop_length"], seed)
        mel = front_end(wave, 4 * H)
        inpaint = tband is not None or fband is not None
        m = oedit.ratio_mask(H, 16, tband, fband) if inpaint else None
        sched = scheds[sname]()
        orders = record_dpm_orders(sched) if sname == "dpm" else None
        record = {}
        s = stand_in(INP if inpaint else I2I, usd, ucfg, mask, sched, ref_vae, record)
        rec = RecordingGenerator(seed)
        kw = dict(prompt=None, image=mel, strength=strength, num_inference_steps=steps, guidance_scale=guidance,
                  generator=rec.g, prompt_embeds=embeds[1:], negative_prompt_embeds=embeds[:1], return_dict=False)
        with recording(rec):
            if inpaint:
                lat_ref = INP.__call__(s, mask_image=m, add_predicted_noise=False, output_type="np", **kw)[0]
            else:
                lat_ref = I2I.__call__(s, output_type="latent", **kw)[0]
        t_ref = time.time() - t0
        eps_post, noise, step_noises = rec.draws[0], rec.draws[1], rec.draws[2:]
        x0 = oedit.latents_from_moments(record["moments"], eps_post, ref_vae.scale_factor)
        trace = []
        t1 = time.time()
        lat_orc = oedit.edit_loop(usd, ucfg, oracle_scheduler(sname), embeds, mask, steps, guidance, strength, x0,
                                  noise, step_noises if sname == "ddpm" else None, inpaint_mask=m, trace=trace)
        t_orc = time.time() - t1
        d = maxdiff(lat_ref, lat_orc)
        t_start = oedit.get_timesteps(steps, strength)
        print(f"{name}: {sname} {steps} steps from t_start {t_start} (strength {strength}), |lat| max "
              f"{float(lat_ref.abs().max()):.3f}, oracle vs reference max diff {d:.3e} (reference {t_ref:.0f} s, oracle "
              f"{t_orc:.0f} s)", flush=True)
        assert d < (1e-4 if unet == "tiny" else 5e-4), d
        n_draws = sum(1 for t in sched.timesteps[t_start:] if int(t) > 0) if sname == "ddpm" else 0
        again = oedit.seeded_draws(seed, tuple(noise.shape), n_draws)
        assert torch.equal(again[0], eps_post) and torch.equal(again[1], noise) and len(again[2]) == len(step_noises)
        assert all(torch.equal(a, b) for a, b in zip(again[2], step_noises))
        x0_key = f"x0_{H}_{seed}"
        if x0_key in out:
            assert np.array_equal(out[x0_key], x0.numpy())
        out[x0_key] = x0.numpy()
        if unet == "tiny":
            out[f"mel_{H}_{seed}"], out[f"moments_{H}_{seed}"] = mel.numpy(), record["moments"].numpy()
        p = f"{name}_"
        out[p + "latents"] = lat_ref.numpy()
        out[p + "step_norms"] = np.asarray([float(x.norm()) for x in trace], dtype=np.float64)
        if m is not None:
            out[p + "mask"] = m.numpy()
        cases[name] = {"unet": unet, "latent_shape": [H, 16], "scheduler": sname, "steps": steps, "strength": strength,
                       "time_band": tband, "freq_band": fband, "guidance": guidance, "seed": seed, "t_start": t_start,
                       "orders": orders, "step_draws": n_draws, "x0_key": x0_key, "latents_max_abs": d}
        if name == DECODED:
            mel_dec = ref_vae.decode_first_stage(lat_ref)
            out[p + "decoded_mel"] = mel_dec.numpy().astype(np.float32)
            out[p + "decoded_wave_i16"] = ref_vae.decode_to_waveform(mel_dec)
    out["cases"] = np.asarray(json.dumps(cases))
    np.savez_compressed(os.path.join(GOLD, "edit.npz"), **out)
    checks.update(cases=cases, strengths=list(STRENGTHS), grid_steps=list(GRID_STEPS),
                  what="text-guided editing / inpainting through the unmodified fork img2img and legacy-inpaint "
                       "pipelines (fp32 CPU); scheduler arithmetic bit-exact, loops to the stated max-abs")
    with open(os.path.join(GOLD, "edit.json"), "w") as f:
        json.dump(checks, f, indent=1, sort_keys=True)
    print(f"tests/golden/edit.npz written ({os.path.getsize(os.path.join(GOLD, 'edit.npz')) / 1e6:.2f} MB) in "
          f"{time.time() - t00:.0f} s")


if __name__ == "__main__":
    main()
