"""Pin oracle.unipc.OracleUniPCMultistep against the UNMODIFIED fork UniPCMultistepScheduler and write
tests/golden/unipc.npz, with what each part measured in tests/golden/unipc.json (TEST INFRASTRUCTURE ONLY; build
container only, a few minutes on 8 cores).

    python -m oracle.make_golden_unipc

Every part asserts oracle == reference (the scheduler loops bit for bit; the UNet loops to UNet round-off, as
make_golden_config1):
  * timestep grids for n in {1, 5, 10, 25};
  * deterministic scheduler loops (the `sin(3x + t/1000)` model on make_golden.py's x0, SD-2.1 betas, 10 steps) over
    order {1, 2, 3} x solver type {bh1, bh2} x predict_x0 {True, False} x prediction {eps, v, sample}, plus
    lower_order_final off, disable_corrector [0] and [0, 2], the midpoint -> bh1 alias, 5- and 25-step runs, and the
    fork's own full loops (test_scheduler_unipc.py:205-215: linear betas, bh1, dummy model and sample);
  * the (corrector, predictor) orders the fork takes at every executed step of loops entered mid-grid;
  * the form of the fork's `einsum("k,bkchw->bchw")` at every shape it ran on here: one term is a plain product, two
    terms are fma(rho_1, D_1, rho_0 * D_0), checked against the fp64 statement of that fma (oracle.unipc.fma32);
  * the unmodified models.AudioDiffusion.inference on the tiny UNet with the fork's UniPC (SD-2.1 config, CFG 3,
    6 steps; conditioning and initial latents of tiny_inference.npz);
  * tiny img2img and legacy-inpaint loops at strength 0.6 through the fork pipelines (make_golden_edit's stand-ins);
  * config 1 at full size (make_golden_config1.inputs()) with UniPC-2 bh2 at 10 steps: final latents and per-step
    latent norms.
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import edit as oedit  # noqa: E402
from oracle import make_golden_config1 as mg1  # noqa: E402
from oracle import make_golden_dpm as mgd  # noqa: E402
from oracle import make_golden_edit as mge  # noqa: E402
from oracle import pipeline as opipe  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle import unipc as ouni  # noqa: E402
from tango_b200 import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SD21 = mgd.SD21
FORK_TEST = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", solver_order=2,
                 solver_type="bh1")
# name: (H, steps, strength, time band, freq band, guidance, seed), the tiny cases of make_golden_edit
EDIT_CASES = {"tiny_unipc": (32, 10, 0.6, None, None, 3.0, 11),
              "tiny_unipc_inpaint": (32, 10, 0.6, (0.25, 0.5), (0.5, 0.75), 3.0, 11)}


def loop_matrix():
    """(scheduler kwargs, steps, model) of every scheduler loop in the golden, in storage order."""
    out = []
    for order in (1, 2, 3):
        for stype in ("bh1", "bh2"):
            for x0p in (True, False):
                for pred in ("epsilon", "v_prediction", "sample"):
                    out.append((dict(SD21, solver_order=order, solver_type=stype, predict_x0=x0p,
                                     prediction_type=pred), 10, "sin"))
    for order in (2, 3):
        out.append((dict(SD21, solver_order=order, prediction_type="epsilon", lower_order_final=False), 10, "sin"))
        for dc in ([0], [0, 2]):
            out.append((dict(SD21, solver_order=order, prediction_type="v_prediction", disable_corrector=dc), 10,
                        "sin"))
    out.append((dict(SD21, solver_order=2, solver_type="midpoint", prediction_type="v_prediction"), 10, "sin"))
    out.append((dict(SD21, solver_order=2, prediction_type="v_prediction"), 5, "sin"))
    out.append((dict(SD21, solver_order=3, solver_type="bh1", prediction_type="epsilon"), 25, "sin"))
    out.append((dict(SD21, solver_order=2, prediction_type="v_prediction"), 25, "sin"))
    for pred in ("epsilon", "v_prediction"):
        out.append((dict(FORK_TEST, prediction_type=pred), 10, "fork"))
    return out


class EinsumCheck:
    """Wraps torch.einsum while the fork runs: every "k,bkchw->bchw" contraction is compared with the kernel's form
    (one term: rho_0 * D_0; two terms: fma(rho_1, D_1, rho_0 * D_0)) and its shape recorded."""

    def __init__(self):
        self.orig = torch.einsum
        self.shapes = {}

    def __call__(self, eq, *ops):
        out = self.orig(eq, *ops)
        if eq == "k,bkchw->bchw":
            rho, D = ops
            if rho.numel() == 1:
                want = rho[0] * D[:, 0]
            else:
                assert rho.numel() == 2
                want = ouni.fma32(rho[1].expand_as(D[:, 1]), D[:, 1], rho[0] * D[:, 0])
            key = f"{rho.numel()}x{tuple(D.shape)}"
            ok, n = self.shapes.get(key, (True, 0))
            self.shapes[key] = (ok and torch.equal(out, want), n + 1)
        return out

    def __enter__(self):
        torch.einsum = self
        return self

    def __exit__(self, *a):
        torch.einsum = self.orig
        return False


def record_orders(sched):
    """Wrap the fork scheduler's UniC / UniP so that each `step` appends its (corrector, predictor) orders."""
    orders, pending = [], {}
    uc, up = sched.multistep_uni_c_bh_update, sched.multistep_uni_p_bh_update

    def c(*a, order, **kw):
        pending["p"] = order
        return uc(*a, order=order, **kw)

    def p(*a, order, **kw):
        orders.append([pending.pop("p", 0), order])
        return up(*a, order=order, **kw)

    sched.multistep_uni_c_bh_update, sched.multistep_uni_p_bh_update = c, p
    return orders


def main():
    torch.set_grad_enabled(False)
    t00 = time.time()
    R = ouni.reference_class()
    gold, checks = {}, {}
    ein = EinsumCheck()

    # ---- the fork's known answers (test_scheduler_unipc.py:205-215)
    known = {}
    for pred, want in (("epsilon", 0.2521), ("v_prediction", 0.1096)):
        x0, fn = mgd.loop_inputs("fork")
        with ein:
            x = mgd.run_loop(R(**dict(FORK_TEST, prediction_type=pred)), 10, x0, fn)
        known[pred] = float(x.abs().mean())
        assert abs(known[pred] - want) < 1e-3, (pred, known[pred])
    checks["fork_known_answers_mean_abs"] = known
    print("fork known answers:", known)

    # ---- timestep grids
    for n in (1, 5, 10, 25):
        r, o = R(**SD21), ouni.OracleUniPCMultistep(**SD21)
        r.set_timesteps(n)
        o.set_timesteps(n)
        assert torch.equal(r.timesteps, o.timesteps) and r.timesteps.dtype == torch.int64
        gold[f"timesteps_{n}"] = r.timesteps.numpy()

    # ---- scheduler loops
    mat = loop_matrix()
    for k, (kw, steps, model) in enumerate(mat):
        x0, fn = mgd.loop_inputs(model)
        with ein:
            xr = mgd.run_loop(R(**kw), steps, x0, fn)
        xo = mgd.run_loop(ouni.OracleUniPCMultistep(**kw), steps, x0, fn)
        assert torch.equal(xr, xo), f"loop {k} {kw} {steps}: oracle not bit-exact"
        gold[f"loop_{k}"] = xr.numpy()
    gold["loop_configs"] = np.array(json.dumps([[kw, steps, model] for kw, steps, model in mat]))
    gold["sin_x0"] = mgd.loop_inputs("sin")[0].numpy()
    checks["loops"] = f"{len(mat)} loops, oracle == reference bit-exact"
    print(f"{len(mat)} scheduler loops: oracle == fork bit for bit ({time.time() - t00:.0f} s)", flush=True)

    # ---- (corrector, predictor) orders of loops entered mid-grid
    orders = {}
    for order in (1, 2, 3):
        for n in (5, 10, 25):
            for st in (0.3, 0.6, 1.0):
                for dc in ([], [0, 2]):
                    s = R(**SD21, solver_order=order, disable_corrector=dc)
                    s.set_timesteps(n)
                    rec = record_orders(s)
                    x = torch.zeros(1, 1, 2, 2)
                    for t in s.timesteps[oedit.get_timesteps(n, st):]:
                        x = s.step(torch.zeros_like(x), t, x).prev_sample
                    orders[f"{order}_{n}_{st}_{dc}"] = rec
    gold["orders"] = np.asarray(json.dumps(orders))

    # ---- tiny AudioDiffusion.inference, UniPC-2 bh2 (the defaults) on the SD-2.1 v-prediction config
    refmod = refshim.audio_diffusion_module()
    U = refshim.unet_class()
    cfg = dict(synth.TINY_UNET_CONFIG)
    sd = synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0)
    ref_unet = U.from_config(dict(cfg)).eval()
    ref_unet.load_state_dict(sd, strict=True)
    ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    embeds, bmask, lat0 = (torch.from_numpy(ti[k]) for k in ("embeds", "mask", "lat0"))
    kw = dict(SD21, prediction_type="v_prediction")
    steps, guidance = 6, 3.0
    with ein:
        lat_ref = refmod.AudioDiffusion.inference(mgd_stub(ref_unet, embeds, bmask, lat0), ["synthetic prompt"],
                                                  R(**kw), steps, guidance, 1, True)
    lat_orc = opipe.inference(sd, cfg, ouni.OracleUniPCMultistep(**kw), embeds, bmask, steps, guidance, lat0)
    d = mg1.maxdiff(lat_ref, lat_orc)
    print(f"tiny inference, UniPC-2 bh2, {steps} steps, CFG {guidance}: oracle-vs-reference {d:.3e}", flush=True)
    assert d < 2e-4
    gold["tiny_latents"] = lat_ref.numpy()
    checks["tiny_inference"] = {"latents_max_abs": d, "steps": steps, "guidance": guidance, "scheduler": kw}
    del ref_unet

    # ---- tiny img2img / legacy inpaint through the fork pipelines
    I2I, INP = mge.import_pipelines()
    A = refshim.autoencoder_class()
    ref_vae = A(**synth.VAE_CONFIG).eval()
    vsd = synth.synth_state_dict(dict(synth.vae_decoder_param_shapes(), **synth.vae_encoder_param_shapes()), seed=0)
    full = ref_vae.state_dict()
    full.update(vsd)
    ref_vae.load_state_dict(full, strict=True)
    emask = torch.from_numpy(ti["mask"])
    edits = {}
    for name, (H, steps, strength, tband, fband, guidance, seed) in EDIT_CASES.items():
        wave = oedit.input_wave(4 * H * synth.STFT_CONFIG["hop_length"], seed)
        mel = mge.front_end(wave, 4 * H)
        inpaint = tband is not None or fband is not None
        m = oedit.ratio_mask(H, 16, tband, fband) if inpaint else None
        sched = R(**kw)
        rec_orders = record_orders(sched)
        record = {}
        s = mge.stand_in(INP if inpaint else I2I, sd, cfg, emask, sched, ref_vae, record)
        rec = mge.RecordingGenerator(seed)
        call = dict(prompt=None, image=mel, strength=strength, num_inference_steps=steps, guidance_scale=guidance,
                    generator=rec.g, prompt_embeds=embeds[1:], negative_prompt_embeds=embeds[:1], return_dict=False)
        with mge.recording(rec), ein:
            if inpaint:
                lat_ref = INP.__call__(s, mask_image=m, add_predicted_noise=False, output_type="np", **call)[0]
            else:
                lat_ref = I2I.__call__(s, output_type="latent", **call)[0]
        eps_post, noise = rec.draws[0], rec.draws[1]
        assert len(rec.draws) == 2          # nothing is drawn after the add-noise draw
        x0 = oedit.latents_from_moments(record["moments"], eps_post, ref_vae.scale_factor)
        trace = []
        lat_orc = oedit.edit_loop(sd, cfg, ouni.OracleUniPCMultistep(**kw), embeds, emask, steps, guidance, strength,
                                  x0, noise, None, inpaint_mask=m, trace=trace)
        d = mg1.maxdiff(lat_ref, lat_orc)
        t_start = oedit.get_timesteps(steps, strength)
        print(f"{name}: UniPC-2 bh2 {steps} steps from t_start {t_start}, oracle vs reference {d:.3e}", flush=True)
        assert d < 1e-4, d
        again = oedit.seeded_draws(seed, tuple(noise.shape), 0)
        assert torch.equal(again[0], eps_post) and torch.equal(again[1], noise)
        gold[f"{name}_x0"] = x0.numpy()
        gold[f"{name}_latents"] = lat_ref.numpy()
        gold[f"{name}_step_norms"] = np.asarray([float(x.norm()) for x in trace], dtype=np.float64)
        if m is not None:
            gold[f"{name}_mask"] = m.numpy()
        edits[name] = {"latent_shape": [H, 16], "steps": steps, "strength": strength, "time_band": tband,
                       "freq_band": fband, "guidance": guidance, "seed": seed, "t_start": t_start,
                       "orders": rec_orders, "latents_max_abs": d}
    gold["edit_cases"] = np.asarray(json.dumps(edits))
    checks["edit"] = edits

    # ---- config 1 at full size, UniPC-2 bh2 at 10 steps
    cfg1, emb1, mask1, lat1, _ = mg1.inputs()
    sd1 = synth.synth_state_dict(synth.unet_param_shapes(cfg1), seed=mg1.SEEDS["weights"])
    ref_unet = U.from_config(dict(cfg1)).eval()
    ref_unet.load_state_dict(sd1, strict=True)
    steps = 10
    r = R(**kw)
    norms = []
    step0 = r.step

    def rec_step(*a, _step=step0, **k):
        out = _step(*a, **k)
        norms.append(float(out.prev_sample.norm()))
        return out

    r.step = rec_step
    t0 = time.time()
    with ein:
        lat_ref = refmod.AudioDiffusion.inference(mgd_stub(ref_unet, emb1, mask1, lat1), ["synthetic prompt"], r, steps,
                                                  mg1.GUIDANCE, 1, True)
    t_ref = time.time() - t0
    trace = []
    lat_orc = opipe.inference(sd1, cfg1, ouni.OracleUniPCMultistep(**kw), emb1, mask1, steps, mg1.GUIDANCE, lat1,
                              trace=trace)
    d = mg1.maxdiff(lat_ref, lat_orc)
    dn = max(abs(a - float(b.norm())) / a for a, b in zip(norms, trace))
    print(f"config-1 UniPC-2 bh2, {steps} steps: |lat| max {lat_ref.abs().max():.3f}, oracle-vs-reference {d:.3e}, "
          f"norms rel {dn:.1e} (reference {t_ref:.0f} s)", flush=True)
    assert d < 5e-4 and dn < 1e-5
    gold[f"config1_latents_{steps}"] = lat_ref.numpy()
    gold[f"config1_step_norms_{steps}"] = np.asarray(norms, dtype=np.float64)
    gold[f"config1_timesteps_{steps}"] = r.timesteps.numpy()
    checks["config1"] = {str(steps): {"latents_max_abs": d, "reference_s": round(t_ref, 1)}, "guidance": mg1.GUIDANCE,
                         "seeds": mg1.SEEDS, "scheduler": kw}

    # ---- the einsum form, at every shape the fork contracted here
    bad = [k for k, (ok, _) in ein.shapes.items() if not ok]
    assert not bad, f"einsum differs from the kernel's form at {bad}"
    checks["einsum"] = {"one_term": "rho_0 * D_0", "two_terms": "fma(rho_1, D_1, rho_0 * D_0)",
                        "holds_at": {k: n for k, (_, n) in sorted(ein.shapes.items())}}
    print("einsum form holds at", sorted(ein.shapes))

    np.savez_compressed(os.path.join(GOLD, "unipc.npz"), **gold)
    checks = dict(checks, torch=torch.__version__,
                  what="fork UniPCMultistepScheduler (scheduling_unipc_multistep.py) through the unmodified reference, "
                       "fp32 CPU")
    with open(os.path.join(GOLD, "unipc.json"), "w") as f:
        json.dump(checks, f, indent=1)
    print(f"wrote {os.path.join(GOLD, 'unipc.npz')} "
          f"({os.path.getsize(os.path.join(GOLD, 'unipc.npz')) / 1e6:.2f} MB) in {time.time() - t00:.0f} s")


def mgd_stub(unet, emb, mask, l0):
    """The `self` of models.AudioDiffusion.inference (as make_golden_dpm): the UNet, fixed conditioning and latents."""
    class _Stub:
        pass

    s = _Stub()
    s.unet, s.set_from = unet, "random"
    s.text_encoder = _Stub()
    s.text_encoder.device = torch.device("cpu")
    s.encode_text_classifier_free = lambda prompt, n: (emb, mask)
    s.prepare_latents = lambda bs, sch, ch, dt, dev: l0 * sch.init_noise_sigma
    return s


if __name__ == "__main__":
    main()
