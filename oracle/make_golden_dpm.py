"""Pin oracle.dpm_solver.OracleDPMSolverMultistep against the UNMODIFIED fork DPMSolverMultistepScheduler and write
tests/golden/dpm_solver.npz, with what each part measured in tests/golden/dpm_solver.json (TEST INFRASTRUCTURE ONLY;
build container only, ~5 min on 8 cores).

    python -m oracle.make_golden_dpm

Every part asserts oracle == reference bit for bit (the full-size loop: to UNet round-off, as make_golden_config1):
  * timestep grids for n in {1, 10, 14, 15, 25};
  * deterministic scheduler loops (the `sin(3x + t/1000)` model on make_golden.py's x0, SD-2.1 betas, 10 steps) over
    order {1, 2, 3} x algorithm {dpmsolver, dpmsolver++} x solver type {midpoint, heun} x prediction {eps, v}, plus
    lower_order_final off, `sample` prediction, the deis / bh2 aliases, 25-step runs (past the < 15 rule) and the
    fork's own full loops (test_scheduler_dpm_multi.py:97-210: linear betas, dummy model and sample);
  * the unmodified models.AudioDiffusion.inference on the tiny UNet with the fork's scheduler (SD-2.1 config, CFG 3,
    6 steps; conditioning and initial latents of tiny_inference.npz);
  * config 1 at full size (make_golden_config1.inputs(): base UNet, 1 prompt, CFG 3, 256 x 16) with DPM-Solver++ 2M
    at 10 and 25 steps: final latents and per-step latent norms.
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

from oracle import dpm_solver as odpm  # noqa: E402
from oracle import make_golden_config1 as mg1  # noqa: E402
from oracle import pipeline as opipe  # noqa: E402
from oracle import refshim  # noqa: E402
from tango_b200 import synth  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
SD21 = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear")
FORK_TEST = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 lower_order_final=False)


def loop_matrix():
    """(scheduler kwargs, steps, model) of every scheduler loop in the golden, in storage order."""
    out = []
    for order in (1, 2, 3):
        for algo in ("dpmsolver", "dpmsolver++"):
            for stype in ("midpoint", "heun"):
                for pred in ("epsilon", "v_prediction"):
                    out.append((dict(SD21, solver_order=order, algorithm_type=algo, solver_type=stype,
                                     prediction_type=pred), 10, "sin"))
    for order in (2, 3):
        out.append((dict(SD21, solver_order=order, prediction_type="epsilon", lower_order_final=False), 10, "sin"))
    for algo in ("dpmsolver", "dpmsolver++"):
        out.append((dict(SD21, solver_order=2, algorithm_type=algo, prediction_type="sample"), 10, "sin"))
    out.append((dict(SD21, solver_order=3, algorithm_type="deis", solver_type="bh2", prediction_type="epsilon"), 10,
                "sin"))
    out.append((dict(SD21, solver_order=2, prediction_type="v_prediction"), 25, "sin"))
    out.append((dict(SD21, solver_order=3, solver_type="heun", prediction_type="epsilon"), 25, "sin"))
    for pred in ("epsilon", "v_prediction"):
        out.append((dict(FORK_TEST, solver_order=2, prediction_type=pred), 10, "fork"))
    return out


def loop_inputs(model: str):
    """(x0, model_fn) of a scheduler loop: make_golden.py section 2, or the fork's dummy sample / model."""
    if model == "sin":
        g = torch.Generator().manual_seed(3)
        return torch.randn(2, 8, 16, 16, generator=g), lambda x, t: torch.sin(x * 3.0 + float(t) / 1000)
    n = 4 * 3 * 8 * 8
    x0 = (torch.arange(n).reshape(3, 8, 8, 4) / n).permute(3, 0, 1, 2).contiguous()   # dummy_sample_deter
    return x0, lambda x, t: x * t / (t + 1)                                           # dummy_model


def run_loop(sched, steps, x0, model):
    sched.set_timesteps(steps)
    x = x0.clone()
    for t in sched.timesteps:
        x = sched.step(model(x, t), t, x)
        x = x.prev_sample if hasattr(x, "prev_sample") else x
    return x


def main():
    torch.set_grad_enabled(False)
    t00 = time.time()
    R = odpm.reference_class()
    gold, checks = {}, {}

    # ---- timestep grids
    for n in (1, 10, 14, 15, 25):
        r, o = R(**SD21), odpm.OracleDPMSolverMultistep(**SD21)
        r.set_timesteps(n)
        o.set_timesteps(n)
        assert torch.equal(r.timesteps, o.timesteps) and r.timesteps.dtype == torch.int64
        gold[f"timesteps_{n}"] = r.timesteps.numpy()
    print("timesteps 25:", gold["timesteps_25"].tolist())

    # ---- scheduler loops
    mat = loop_matrix()
    for k, (kw, steps, model) in enumerate(mat):
        x0, fn = loop_inputs(model)
        xr = run_loop(R(**kw), steps, x0, fn)
        xo = run_loop(odpm.OracleDPMSolverMultistep(**kw), steps, x0, fn)
        assert torch.equal(xr, xo), f"loop {k} {kw} {steps}: oracle not bit-exact"
        gold[f"loop_{k}"] = xr.numpy()
        if model == "fork":
            print(f"fork full loop {kw['prediction_type']}: mean |x| = {float(xr.abs().mean()):.4f}")
    gold["loop_configs"] = np.array(json.dumps([[kw, steps, model] for kw, steps, model in mat]))
    gold["sin_x0"] = loop_inputs("sin")[0].numpy()
    checks["loops"] = f"{len(mat)} loops, oracle == reference bit-exact"

    # ---- tiny AudioDiffusion.inference
    refmod = refshim.audio_diffusion_module()
    U = refshim.unet_class()
    cfg = dict(synth.TINY_UNET_CONFIG)
    sd = synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0)
    ref_unet = U.from_config(dict(cfg)).eval()
    ref_unet.load_state_dict(sd, strict=True)
    ti = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    embeds, bmask, lat0 = (torch.from_numpy(ti[k]) for k in ("embeds", "mask", "lat0"))
    kw = dict(SD21, prediction_type="v_prediction")

    class _Stub:
        pass

    def stub_for(unet, emb, mask, l0):
        s = _Stub()
        s.unet, s.set_from = unet, "random"
        s.text_encoder = _Stub()
        s.text_encoder.device = torch.device("cpu")
        s.encode_text_classifier_free = lambda prompt, n: (emb, mask)
        s.prepare_latents = lambda bs, sch, ch, dt, dev: l0 * sch.init_noise_sigma
        return s

    steps, guidance = 6, 3.0
    lat_ref = refmod.AudioDiffusion.inference(stub_for(ref_unet, embeds, bmask, lat0), ["synthetic prompt"], R(**kw),
                                              steps, guidance, 1, True)
    lat_orc = opipe.inference(sd, cfg, odpm.OracleDPMSolverMultistep(**kw), embeds, bmask, steps, guidance, lat0)
    d = mg1.maxdiff(lat_ref, lat_orc)
    print(f"tiny inference, DPM-Solver++ 2M, {steps} steps, CFG {guidance}: oracle-vs-reference {d:.3e}")
    assert d < 2e-4
    gold["tiny_latents"] = lat_ref.numpy()
    checks["tiny_inference"] = {"latents_max_abs": d, "steps": steps, "guidance": guidance}
    del ref_unet

    # ---- config 1 at full size
    cfg1, emb1, mask1, lat1, _ = mg1.inputs()
    sd1 = synth.synth_state_dict(synth.unet_param_shapes(cfg1), seed=mg1.SEEDS["weights"])
    ref_unet = U.from_config(dict(cfg1)).eval()
    ref_unet.load_state_dict(sd1, strict=True)
    full = {}
    for steps in (10, 25):
        r = R(**kw)
        norms = []
        step0 = r.step

        def rec(*a, _step=step0, **k):
            out = _step(*a, **k)
            norms.append(float(out.prev_sample.norm()))
            return out

        r.step = rec
        t0 = time.time()
        lat_ref = refmod.AudioDiffusion.inference(stub_for(ref_unet, emb1, mask1, lat1), ["synthetic prompt"], r, steps,
                                                  mg1.GUIDANCE, 1, True)
        t_ref = time.time() - t0
        trace = []
        lat_orc = opipe.inference(sd1, cfg1, odpm.OracleDPMSolverMultistep(**kw), emb1, mask1, steps, mg1.GUIDANCE,
                                  lat1, trace=trace)
        d = mg1.maxdiff(lat_ref, lat_orc)
        dn = max(abs(a - float(b.norm())) / a for a, b in zip(norms, trace))
        print(f"config-1 DPM-Solver++ 2M, {steps} steps: |lat| max {lat_ref.abs().max():.3f}, oracle-vs-reference "
              f"{d:.3e}, norms rel {dn:.1e} (reference {t_ref:.0f} s)", flush=True)
        assert d < 5e-4 and dn < 1e-5
        gold[f"config1_latents_{steps}"] = lat_ref.numpy()
        gold[f"config1_step_norms_{steps}"] = np.asarray(norms, dtype=np.float64)
        gold[f"config1_timesteps_{steps}"] = r.timesteps.numpy()
        full[steps] = {"latents_max_abs": d, "reference_s": round(t_ref, 1)}
    checks["config1"] = dict(full, guidance=mg1.GUIDANCE, seeds=mg1.SEEDS, scheduler=kw)

    np.savez_compressed(os.path.join(GOLD, "dpm_solver.npz"), **gold)
    checks = dict(checks, generated=time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime()), torch=torch.__version__,
                  what="fork DPMSolverMultistepScheduler (scheduling_dpmsolver_multistep.py) through the unmodified "
                       "reference, fp32 CPU")
    with open(os.path.join(GOLD, "dpm_solver.json"), "w") as f:
        json.dump(checks, f, indent=1)
    print(f"wrote {os.path.join(GOLD, 'dpm_solver.npz')} "
          f"({os.path.getsize(os.path.join(GOLD, 'dpm_solver.npz')) / 1e6:.2f} MB) in {time.time() - t00:.0f} s")


if __name__ == "__main__":
    main()
