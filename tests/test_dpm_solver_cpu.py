"""CPU: the multistep DPM-Solver(++) scheduler. The oracle is pinned to the fork's known answers and to
tests/golden/dpm_solver.npz; the product's coefficient tables and its inference loop are driven through a torch
statement of what tng_dpm_step computes (cabi_spec.spec_dpm_step) and must reproduce the reference bit for bit. Nothing
here is a CPU fallback of the product: the substitution exists only under pytest's monkeypatch."""
import json
import os

import numpy as np
import pytest
import torch

import cabi_spec
from oracle import dpm_solver as odpm
from oracle import schedulers as osched
from tango_b200 import lib as L
from tango_b200 import synth
from tango_b200.schedulers import DDPMScheduler, DPMSolverMultistepScheduler

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CPU = torch.device("cpu")
FORK_TEST = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 lower_order_final=False, solver_order=2)


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
    return np.load(os.path.join(GOLD, "dpm_solver.npz"))


def golden_loops():
    gd = golden()
    return gd, json.loads(str(gd["loop_configs"]))


def loop_inputs(model):
    """The x0 / model of oracle/make_golden_dpm.py's scheduler loops."""
    if model == "sin":
        return torch.from_numpy(golden()["sin_x0"]), lambda x, t: torch.sin(x * 3.0 + float(t) / 1000)
    n = 4 * 3 * 8 * 8
    x0 = (torch.arange(n).reshape(3, 8, 8, 4) / n).permute(3, 0, 1, 2).contiguous()
    return x0, lambda x, t: x * t / (t + 1)


def run_loop(sched, steps, x0, model):
    sched.set_timesteps(steps)
    x = x0.clone()
    for t in sched.timesteps:
        out = sched.step(model(x, t), t, x)
        x = out.prev_sample if hasattr(out, "prev_sample") else out
    return x


# ---------------------------------------------------------------------------------------------------------- oracle
def test_oracle_meets_fork_known_answers():
    """test_scheduler_dpm_multi.py:194-210 (mean |x| 0.3301 for epsilon, 0.2251 for v-prediction) and the 25-step
    SD-2.1 grid."""
    for pred, want in (("epsilon", 0.3301), ("v_prediction", 0.2251)):
        x0, model = loop_inputs("fork")
        x = run_loop(odpm.OracleDPMSolverMultistep(**dict(FORK_TEST, prediction_type=pred)), 10, x0, model)
        assert abs(float(x.abs().mean()) - want) < 1e-3
    o = odpm.OracleDPMSolverMultistep(**osched.SD21_CONFIG)
    o.set_timesteps(25)
    ts = o.timesteps.tolist()
    assert ts[:2] == [999, 959] and ts[-1] == 40 and len(ts) == 25


def test_oracle_equals_golden_bit_for_bit():
    gd, mat = golden_loops()
    assert len(mat) >= 24
    for n in (1, 10, 14, 15, 25):
        o = odpm.OracleDPMSolverMultistep(**osched.SD21_CONFIG)
        o.set_timesteps(n)
        assert o.timesteps.tolist() == gd[f"timesteps_{n}"].tolist()
    for k, (kw, steps, model) in enumerate(mat):
        x0, fn = loop_inputs(model)
        x = run_loop(odpm.OracleDPMSolverMultistep(**kw), steps, x0, fn)
        assert np.array_equal(x.numpy(), gd[f"loop_{k}"]), (k, kw, steps)


# ---------------------------------------------------------------------------------------------------------- product
def test_product_timesteps_and_orders():
    gd = golden()
    s = DPMSolverMultistepScheduler.from_pretrained()
    for n in (1, 10, 14, 15, 25):
        s.set_timesteps(n)
        assert s.timesteps.dtype == torch.int64 and s.timesteps.tolist() == gd[f"timesteps_{n}"].tolist()
    s3 = DPMSolverMultistepScheduler.from_pretrained(solver_order=3)
    s3.set_timesteps(10)     # < 15 steps: the last two steps drop to order 1 and 2
    assert [s3.order_at(i) for i in range(10)] == [1, 2, 3, 3, 3, 3, 3, 3, 2, 1]
    s3.set_timesteps(15)
    assert [s3.order_at(i) for i in range(15)] == [1, 2] + [3] * 13
    assert s3.coefficient_table().shape == (15, 11)


def test_product_tables_reproduce_every_golden_loop(spec_backend):
    """DPMSolverMultistepScheduler.step, i.e. the host coefficient rows + history bookkeeping fed to the tng_dpm_step
    arithmetic, equals the fork's loops bit for bit, over the whole supported matrix."""
    gd, mat = golden_loops()
    for k, (kw, steps, model) in enumerate(mat):
        x0, fn = loop_inputs(model)
        s = DPMSolverMultistepScheduler(**kw)
        x = run_loop(s, steps, x0, fn)
        assert np.array_equal(x.numpy(), gd[f"loop_{k}"]), (k, kw, steps)
        assert s.lower_order_nums == kw["solver_order"] and len(s.model_outputs) == kw["solver_order"]


def test_product_step_tracks_lower_order_nums_like_the_reference(spec_backend):
    """`step` called step by step keeps the reference's `lower_order_nums` / `model_outputs`: a second loop over the same
    grid without `set_timesteps` starts at order 3 (the rows then come from the out-of-sequence path)."""
    x0, fn = loop_inputs("sin")
    kw = dict(osched.SD21_CONFIG, solver_order=3, prediction_type="epsilon")
    p, o = DPMSolverMultistepScheduler.from_config(kw), odpm.OracleDPMSolverMultistep(**kw)
    xp, xo = run_loop(p, 6, x0, fn), run_loop(o, 6, x0, fn)
    for t in p.timesteps[:3]:           # continue with the stale history, as the reference does
        xp = p.step(fn(xp, t), t, xp).prev_sample
        xo = o.step(fn(xo, t), t, xo)
    assert np.array_equal(xp.numpy(), xo.numpy())
    # a timestep outside the grid takes the last index with its own timestep (:458-463)
    yp = p.step(fn(xp, 500), 500, xp).prev_sample
    yo = o.step(fn(xo, torch.tensor(500)), torch.tensor(500), xo)
    assert np.array_equal(yp.numpy(), yo.numpy())


def test_from_config_and_refusals():
    ddpm = DDPMScheduler.from_pretrained()
    s = DPMSolverMultistepScheduler.from_config(ddpm.config)
    assert s.config["prediction_type"] == "v_prediction" and s.config["solver_order"] == 2
    assert s.config["beta_schedule"] == "scaled_linear" and "variance_type" not in s.config
    assert torch.equal(s.alphas_cumprod, ddpm.alphas_cumprod)
    assert s.order == 1 and s.init_noise_sigma == 1.0
    x = torch.ones(2)
    assert s.scale_model_input(x, 3) is x
    assert DPMSolverMultistepScheduler(algorithm_type="deis", solver_type="bh1").config["algorithm_type"] == "dpmsolver++"
    with pytest.raises(NotImplementedError):
        DPMSolverMultistepScheduler(thresholding=True)
    with pytest.raises(NotImplementedError):
        DPMSolverMultistepScheduler(beta_schedule="squaredcos_cap_v2")
    with pytest.raises(NotImplementedError):
        DPMSolverMultistepScheduler(algorithm_type="unipc")
    with pytest.raises(ValueError):
        DPMSolverMultistepScheduler.from_pretrained("some/hub-name")
    with pytest.raises(ValueError):
        DPMSolverMultistepScheduler().step(torch.zeros(1, 1, 1, 1), 1, torch.zeros(1, 1, 1, 1))


def test_from_pretrained_reads_local_scheduler_config(tmp_path):
    d = tmp_path / "scheduler"
    d.mkdir()
    (d / "scheduler_config.json").write_text(json.dumps(dict(osched.SD21_CONFIG, prediction_type="epsilon",
                                                             _class_name="DDPMScheduler", variance_type="fixed_small")))
    s = DPMSolverMultistepScheduler.from_pretrained(str(tmp_path), subfolder="scheduler", solver_order=3)
    assert s.config["prediction_type"] == "epsilon" and s.config["solver_order"] == 3


@pytest.mark.parametrize("precision,tol", [("split", 1e-4), ("bf16", 6e-2)])
def test_inference_loop_orchestration_vs_reference_golden(spec_backend, precision, tol):
    """AudioDiffusion.inference with the DPM-Solver++ 2M scheduler (CFG, per-step tng_dpm_step with rotating history
    slots) against the fork's scheduler in the unmodified reference loop (tiny UNet, CFG 3, 6 steps)."""
    from tango_b200.pipeline import AudioDiffusion
    gd, ti = golden(), np.load(os.path.join(GOLD, "tiny_inference.npz"))
    cfg = synth.TINY_UNET_CONFIG
    m = AudioDiffusion(unet_config=cfg, precision=precision, use_cuda_graph=False).to(CPU)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    sch = DPMSolverMultistepScheduler.from_config(DDPMScheduler.from_pretrained().config)
    calls = []
    orig = L.dpm_step
    L.dpm_step = lambda *a, **k: (calls.append(a[5]), orig(*a, **k))[1]
    try:
        trace = []
        lat = m.inference(["synthetic prompt"], sch, 6, 3.0, prompt_embeds=torch.from_numpy(ti["embeds"]),
                          boolean_prompt_mask=torch.from_numpy(ti["mask"]), latents=torch.from_numpy(ti["lat0"]),
                          latent_shape=(32, 16), trace=trace)
    finally:
        L.dpm_step = orig
    assert calls == [1, 2, 2, 2, 2, 1] and len(trace) == 6      # lower_order_final: the last of < 15 steps is order 1
    e = float((lat.double() - torch.from_numpy(gd["tiny_latents"]).double()).norm()
              / torch.from_numpy(gd["tiny_latents"]).double().norm())
    assert e < tol, e


def test_advance_rng_draws_only_the_initial_latents(spec_backend):
    from tango_b200.pipeline import AudioDiffusion
    m = AudioDiffusion(unet_config=synth.TINY_UNET_CONFIG, precision="split", use_cuda_graph=False).to(CPU)
    g = torch.Generator().manual_seed(5)
    m.advance_rng(3, DPMSolverMultistepScheduler.from_pretrained(), 20, g, latent_shape=(32, 16))
    g2 = torch.Generator().manual_seed(5)
    torch.randn(3, 8, 32, 16, generator=g2)
    assert torch.equal(torch.randn(4, generator=g), torch.randn(4, generator=g2))


def test_cli_dpmsolver_path_on_synthetic_tiny(spec_backend, tmp_path, monkeypatch):
    """`--scheduler dpmsolver++ --solver_order 3` builds the DPM-Solver on the checkpoint's scheduler config and the
    summary line records it (generation itself stubbed)."""
    from tango_b200 import cli
    from tango_b200.pipeline import Tango
    man = tmp_path / "p.json"
    man.write_text("\n".join(json.dumps({"captions": f"prompt {i}"}) for i in range(3)))
    seen = []

    def fake_generate(self, prompts, steps, guidance, batch_size, **kw):
        seen.append(self.scheduler)
        return [np.zeros(1600, dtype=np.int16) for _ in prompts]

    monkeypatch.setattr(Tango, "generate_for_batch", fake_generate)
    res = cli.main(["--checkpoint", "synthetic:tiny", "--device", "cpu", "--test_file", str(man), "--num_steps", "20",
                    "--scheduler", "dpmsolver++", "--solver_order", "3", "--output_root", str(tmp_path / "o"),
                    "--exp_id", "x", "--precision", "split"])
    assert isinstance(seen[0], DPMSolverMultistepScheduler)
    sc = res["scheduler_config"]
    assert sc["solver_order"] == 3 and sc["algorithm_type"] == "dpmsolver++" and sc["prediction_type"] == "v_prediction"
    line = json.loads((tmp_path / "o" / "tango_checkpoint_summary.jsonl").read_text().strip())
    assert line["scheduler_config"]["solver_order"] == 3 and line["args"]["scheduler"] == "dpmsolver++"
    t = Tango.from_synthetic(synth.TINY_UNET_CONFIG, device="cpu", precision="split", scheduler="dpmsolver++")
    assert isinstance(t.scheduler, DPMSolverMultistepScheduler) and t.scheduler.config["solver_order"] == 2


def test_tango_generate_for_batch_with_dpm_scheduler(spec_backend):
    """`tango.scheduler = DPMSolverMultistepScheduler.from_config(tango.scheduler.config)` then generate_for_batch: the
    latents equal the oracle DPM-Solver++ loop on the same conditioning."""
    from oracle import pipeline as opipe
    from tango_b200.pipeline import Tango
    cfg = synth.TINY_UNET_CONFIG
    t = Tango.from_synthetic(unet_config=cfg, device="cpu", precision="split")
    t.model.use_cuda_graph = False
    t.scheduler = DPMSolverMultistepScheduler.from_config(t.scheduler.config)
    prompts = ["a dog barking in the rain", "church bells"]
    lat0, _ = synth.synth_noise(2, 0, shape=(8, 32, 16), seed=11)
    got = {}
    orig = t._decode
    t._decode = lambda lat: (got.setdefault("lat", lat.clone()), orig(lat))[1]
    waves = t.generate_for_batch(prompts, steps=4, guidance=3, batch_size=2, latent_shape=(32, 16), latents=lat0)
    assert len(waves) == 2 and all(w.dtype == np.int16 for w in waves)
    pe, pm = t.model.encode_text_classifier_free(prompts, 1)
    usd = synth.synth_state_dict(synth.unet_param_shapes(cfg), 0)
    want = opipe.inference(usd, cfg, odpm.OracleDPMSolverMultistep(**osched.SD21_CONFIG), pe, pm, 4, 3.0, lat0)
    e = float((got["lat"].double() - want.double()).norm() / want.double().norm())
    assert e < 1e-4, e
