"""CPU: the multistep UniPC scheduler. The oracle is pinned to the fork's known answers and to tests/golden/unipc.npz;
the product's coefficient rows, its state and its loops are driven through a torch statement of what tng_unipc_step
computes (unipc_spec.spec_unipc_step) and must reproduce the reference bit for bit. Nothing here is a CPU fallback of the
product: the substitution exists only under pytest's monkeypatch."""
import json
import os

import numpy as np
import pytest
import torch

import unipc_spec
from oracle import edit as oedit
from oracle import schedulers as osched
from oracle import unipc as ouni
from tango_b200 import lib as L
from tango_b200 import synth
from tango_b200.schedulers import DDPMScheduler, DPMSolverMultistepScheduler, UniPCMultistepScheduler

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CPU = torch.device("cpu")
FORK_TEST = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", solver_order=2,
                 solver_type="bh1")


@pytest.fixture
def spec_backend(monkeypatch):
    unipc_spec.install_unipc_spec_backend(monkeypatch)

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
    return np.load(os.path.join(GOLD, "unipc.npz"))


def loop_inputs(model):
    """The x0 / model of oracle/make_golden_unipc.py's scheduler loops."""
    if model == "sin":
        return torch.from_numpy(golden()["sin_x0"]), lambda x, t: torch.sin(x * 3.0 + float(t) / 1000)
    n = 4 * 3 * 8 * 8
    x0 = (torch.arange(n).reshape(3, 8, 8, 4) / n).permute(3, 0, 1, 2).contiguous()
    return x0, lambda x, t: x * t / (t + 1)


def run_loop(sched, steps, x0, model, start=0):
    sched.set_timesteps(steps)
    x = x0.clone()
    for t in sched.timesteps[start:]:
        out = sched.step(model(x, t), t, x)
        x = out.prev_sample if hasattr(out, "prev_sample") else out
    return x


def sd21(**kw):
    return UniPCMultistepScheduler.from_config(DDPMScheduler.from_pretrained().config, **kw)


# ---------------------------------------------------------------------------------------------------------- oracle
def test_oracle_meets_fork_known_answers():
    """test_scheduler_unipc.py:205-215: mean |x| 0.2521 for epsilon, 0.1096 for v-prediction."""
    for pred, want in (("epsilon", 0.2521), ("v_prediction", 0.1096)):
        x0, model = loop_inputs("fork")
        x = run_loop(ouni.OracleUniPCMultistep(**dict(FORK_TEST, prediction_type=pred)), 10, x0, model)
        assert abs(float(x.abs().mean()) - want) < 1e-3


def test_oracle_equals_golden_bit_for_bit():
    gd = golden()
    mat = json.loads(str(gd["loop_configs"]))
    assert len(mat) >= 40
    for k, (kw, steps, model) in enumerate(mat):
        x0, fn = loop_inputs(model)
        assert np.array_equal(run_loop(ouni.OracleUniPCMultistep(**kw), steps, x0, fn).numpy(), gd[f"loop_{k}"]), k


def test_fma32_is_one_rounding():
    a, b = torch.tensor([1.0 + 2.0 ** -23]), torch.tensor([1.0 - 2.0 ** -23])
    c = torch.tensor([-1.0])
    assert float(ouni.fma32(a, b, c)) == -(2.0 ** -46)      # a * b rounded first would give 0
    from fractions import Fraction
    g = torch.Generator().manual_seed(0)
    x, y, z = (torch.randn(256, generator=g) * 2.0 ** torch.randint(-20, 20, (256,), generator=g) for _ in range(3))
    got = ouni.fma32(x, y, z)
    for a, b, c, r in zip(x.tolist(), y.tolist(), z.tolist(), got.tolist()):
        exact = Fraction(a) * Fraction(b) + Fraction(c)
        lo, hi = np.nextafter(np.float32(r), np.float32(-np.inf)), np.nextafter(np.float32(r), np.float32(np.inf))
        assert abs(exact - Fraction(r)) <= min(abs(exact - Fraction(float(lo))), abs(exact - Fraction(float(hi))))


# ---------------------------------------------------------------------------------------------------------- product
def test_product_timesteps_and_orders():
    gd = golden()
    s = sd21()
    for n in (1, 5, 10, 25):
        s.set_timesteps(n)
        assert s.timesteps.dtype == torch.int64 and s.timesteps.tolist() == gd[f"timesteps_{n}"].tolist()
    s3 = sd21(solver_order=3)
    s3.set_timesteps(10)     # lower_order_final: the predictor order is at most the number of steps left
    assert [s3.order_at(i) for i in range(10)] == [(0, 1), (1, 2), (2, 3)] + [(3, 3)] * 5 + [(3, 2), (2, 1)]
    assert s3.coefficient_table().shape == (10, 18)
    # every executed step of the fork's mid-grid loops, with and without disable_corrector
    for key, want in json.loads(str(gd["orders"])).items():
        order, n, st, dc = key.split("_")
        s = sd21(solver_order=int(order), disable_corrector=json.loads(dc))
        s.set_timesteps(int(n))
        t_start = oedit.get_timesteps(int(n), float(st))
        s.loop_table(None, t_start)
        assert [list(o) for o in s._loop_orders[t_start:]] == want, key


def test_product_tables_reproduce_every_golden_loop(spec_backend):
    """UniPCMultistepScheduler.step, i.e. the host rows + state fed to the tng_unipc_step arithmetic, equals the fork's
    loops bit for bit over the whole golden matrix; the loop table's rows are the rows `step` uses."""
    gd = golden()
    for k, (kw, steps, model) in enumerate(json.loads(str(gd["loop_configs"]))):
        x0, fn = loop_inputs(model)
        s = UniPCMultistepScheduler(**kw)
        x = run_loop(s, steps, x0, fn)
        assert np.array_equal(x.numpy(), gd[f"loop_{k}"]), (k, kw, steps)
        tab = s.coefficient_table()
        assert all(torch.equal(tab[i], s._coefficients_at(i, s.order_at(i))) for i in range(steps))


def test_product_step_state_tracks_the_reference(spec_backend):
    """`step` keeps the reference's state: a loop reused after `set_timesteps`, a loop continued without it (stale
    history, corrector on), a timestep outside the grid, and a loop entered mid-grid."""
    x0, fn = loop_inputs("sin")
    for kw in (dict(osched.SD21_CONFIG, solver_order=3, prediction_type="epsilon"),
               dict(osched.SD21_CONFIG, solver_order=2, solver_type="bh1", predict_x0=False)):
        p, o = UniPCMultistepScheduler.from_config(kw), ouni.OracleUniPCMultistep(**kw)
        xp, xo = run_loop(p, 6, x0, fn), run_loop(o, 6, x0, fn)
        xp, xo = run_loop(p, 5, xp, fn), run_loop(o, 5, xo, fn)      # reuse after set_timesteps
        assert np.array_equal(xp.numpy(), xo.numpy())
        for t in p.timesteps[:3]:
            xp = p.step(fn(xp, t), t, xp).prev_sample
            xo = o.step(fn(xo, t), t, xo)
        assert np.array_equal(xp.numpy(), xo.numpy())
        yp = p.step(fn(xp, 500), 500, xp).prev_sample
        yo = o.step(fn(xo, torch.tensor(500)), torch.tensor(500), xo)
        assert np.array_equal(yp.numpy(), yo.numpy())
        assert p.lower_order_nums == o.lower_order_nums and p.this_order == o.this_order
        assert np.array_equal(p.last_sample.numpy(), o.last_sample.numpy())
        zp, zo = run_loop(p, 10, x0, fn, start=4), run_loop(o, 10, x0, fn, start=4)
        assert np.array_equal(zp.numpy(), zo.numpy())


def test_from_config_refusals_and_alias():
    dpm = DPMSolverMultistepScheduler.from_pretrained()
    s = UniPCMultistepScheduler.from_config(dpm.config)
    assert s.config["solver_type"] == "bh1"          # dpm.config carries solver_type="midpoint"
    assert s.config["prediction_type"] == "v_prediction" and "algorithm_type" not in s.config
    assert torch.equal(s.alphas_cumprod, dpm.alphas_cumprod) and s.order == 1 and s.init_noise_sigma == 1.0
    for st in ("heun", "logrho"):
        assert UniPCMultistepScheduler(solver_type=st).config["solver_type"] == "bh1"
    assert UniPCMultistepScheduler().config["solver_type"] == "bh2"
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(thresholding=True)
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(solver_p=DDPMScheduler())
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(beta_schedule="squaredcos_cap_v2")
    with pytest.raises(NotImplementedError):
        UniPCMultistepScheduler(solver_type="bh3")
    with pytest.raises(ValueError):
        UniPCMultistepScheduler(solver_order=4)
    with pytest.raises(ValueError):
        UniPCMultistepScheduler().step(torch.zeros(1, 1, 1, 1), 1, torch.zeros(1, 1, 1, 1))


@pytest.mark.parametrize("precision,tol", [("split", 1e-4), ("bf16", 6e-2)])
def test_inference_loop_orchestration_vs_reference_golden(spec_backend, precision, tol):
    """AudioDiffusion.inference with UniPC-2 bh2 (CFG, per-step tng_unipc_step over k + 1 history slots and the
    persistent corrected sample) against the fork's scheduler in the unmodified reference loop (tiny UNet, 6 steps)."""
    from tango_b200.pipeline import AudioDiffusion
    gd, ti = golden(), np.load(os.path.join(GOLD, "tiny_inference.npz"))
    cfg = synth.TINY_UNET_CONFIG
    m = AudioDiffusion(unet_config=cfg, precision=precision, use_cuda_graph=False).to(CPU)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    calls = []
    orig = L.unipc_step
    L.unipc_step = lambda *a, **k: (calls.append((a[5], a[6])), orig(*a, **k))[1]
    try:
        lat = m.inference(["synthetic prompt"], sd21(), 6, 3.0, prompt_embeds=torch.from_numpy(ti["embeds"]),
                          boolean_prompt_mask=torch.from_numpy(ti["mask"]), latents=torch.from_numpy(ti["lat0"]),
                          latent_shape=(32, 16))
    finally:
        L.unipc_step = orig
    assert calls == [(0, 1), (1, 2), (2, 2), (2, 2), (2, 2), (2, 1)]
    want = torch.from_numpy(gd["tiny_latents"]).double()
    e = float((lat.double() - want).norm() / want.norm())
    assert e < tol, e


@pytest.mark.parametrize("case", ["tiny_unipc", "tiny_unipc_inpaint"])
def test_edit_orchestration_vs_golden(spec_backend, case):
    """The edit loop entered mid-grid (no corrector at its first step; the inpaint blend rewrites only the sample)
    against the fork's img2img / legacy-inpaint pipelines."""
    from tango_b200.pipeline import AudioDiffusion
    gd, ti = golden(), np.load(os.path.join(GOLD, "tiny_inference.npz"))
    c = json.loads(str(gd["edit_cases"]))[case]
    cfg = synth.TINY_UNET_CONFIG
    m = AudioDiffusion(unet_config=cfg, precision="split", use_cuda_graph=False).to(CPU)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    x0 = torch.from_numpy(gd[f"{case}_x0"])
    noise = oedit.seeded_draws(c["seed"], tuple(x0.shape), 0)[1]
    mask = torch.from_numpy(gd[f"{case}_mask"]) if f"{case}_mask" in gd else None
    s = sd21()
    lat = m.inference(None, s, c["steps"], c["guidance"], prompt_embeds=torch.from_numpy(ti["embeds"]),
                      boolean_prompt_mask=torch.from_numpy(ti["mask"]), latent_shape=tuple(c["latent_shape"]),
                      init_latents=x0, init_noise=noise, strength=c["strength"], inpaint_mask=mask)
    assert [list(o) for o in s._loop_orders[c["t_start"]:]] == c["orders"]
    want = torch.from_numpy(gd[f"{case}_latents"]).double()
    e = float((lat.double() - want).norm() / want.norm())
    assert e < 1e-4, e


def test_advance_rng_draws_only_the_initial_latents(spec_backend):
    from tango_b200.pipeline import AudioDiffusion
    m = AudioDiffusion(unet_config=synth.TINY_UNET_CONFIG, precision="split", use_cuda_graph=False).to(CPU)
    g = torch.Generator().manual_seed(5)
    m.advance_rng(3, sd21(), 10, g, latent_shape=(32, 16))
    g2 = torch.Generator().manual_seed(5)
    torch.randn(3, 8, 32, 16, generator=g2)
    assert torch.equal(torch.randn(4, generator=g), torch.randn(4, generator=g2))


def test_cli_unipc_path_on_synthetic_tiny(spec_backend, tmp_path, monkeypatch):
    from tango_b200 import cli
    from tango_b200.pipeline import Tango
    man = tmp_path / "p.json"
    man.write_text("\n".join(json.dumps({"captions": f"prompt {i}"}) for i in range(2)))
    seen = []

    def fake_generate(self, prompts, steps, guidance, batch_size, **kw):
        seen.append(self.scheduler)
        return [np.zeros(1600, dtype=np.int16) for _ in prompts]

    monkeypatch.setattr(Tango, "generate_for_batch", fake_generate)
    res = cli.main(["--checkpoint", "synthetic:tiny", "--device", "cpu", "--test_file", str(man), "--num_steps", "10",
                    "--scheduler", "unipc", "--solver_order", "3", "--output_root", str(tmp_path / "o"),
                    "--exp_id", "x", "--precision", "split"])
    assert isinstance(seen[0], UniPCMultistepScheduler)
    sc = res["scheduler_config"]
    assert sc["solver_order"] == 3 and sc["solver_type"] == "bh2" and sc["prediction_type"] == "v_prediction"
    t = Tango.from_synthetic(synth.TINY_UNET_CONFIG, device="cpu", precision="split", scheduler="unipc")
    assert isinstance(t.scheduler, UniPCMultistepScheduler) and t.scheduler.config["solver_order"] == 2
    import tango_b200
    assert tango_b200.UniPCMultistepScheduler is UniPCMultistepScheduler


def test_tango_generate_for_batch_with_unipc(spec_backend):
    from oracle import pipeline as opipe
    from tango_b200.pipeline import Tango
    cfg = synth.TINY_UNET_CONFIG
    t = Tango.from_synthetic(unet_config=cfg, device="cpu", precision="split")
    t.model.use_cuda_graph = False
    t.scheduler = UniPCMultistepScheduler.from_config(t.scheduler.config)
    prompts = ["a dog barking in the rain", "church bells"]
    lat0, _ = synth.synth_noise(2, 0, shape=(8, 32, 16), seed=11)
    got = {}
    orig = t._decode
    t._decode = lambda lat: (got.setdefault("lat", lat.clone()), orig(lat))[1]
    waves = t.generate_for_batch(prompts, steps=4, guidance=3, batch_size=2, latent_shape=(32, 16), latents=lat0)
    assert len(waves) == 2 and all(w.dtype == np.int16 for w in waves)
    pe, pm = t.model.encode_text_classifier_free(prompts, 1)
    usd = synth.synth_state_dict(synth.unet_param_shapes(cfg), 0)
    want = opipe.inference(usd, cfg, ouni.OracleUniPCMultistep(**osched.SD21_CONFIG), pe, pm, 4, 3.0, lat0)
    e = float((got["lat"].double() - want.double()).norm() / want.double().norm())
    assert e < 1e-4, e


def test_unipc_step_rejects_bad_arguments_on_host_buffers():
    """tng_unipc_step refuses, before any CUDA call, orders outside range, missing history or `last`, m_cur aliasing a
    slot it reads, and what every latent update refuses (host pointers: nothing is launched)."""
    lib = L.load()
    buf = [torch.zeros(64) for _ in range(6)]
    mo, smp, coef, mc, h1, h2 = (b.data_ptr() for b in buf)
    last, prev = torch.zeros(64).data_ptr(), torch.zeros(64).data_ptr()

    def call(p=1, q=2, m_cur=mc, hist=(h1, h2, None), last_=last, prev_=prev, ld_mo=8, C=8, mo_=mo):
        return lib.tng_unipc_step(mo_, ld_mo, 0, 1.0, smp, coef, p, q, m_cur, *hist, last_, prev_, None, 0, 0, 1, C, 8,
                                  None)

    cases = {"corrector order": dict(p=4), "predictor order": dict(q=0), "history slot": dict(p=2, hist=(h1, None, None)),
             "aliases": dict(m_cur=h1), "needs last": dict(last_=None), "ld_mo": dict(ld_mo=4),
             "null argument": dict(mo_=None), "bad shape": dict(C=0)}
    for what, kw in cases.items():
        assert call(**kw) != 0, what
        msg = lib.tng_last_error().decode()
        assert "unipc_step" in msg and what in msg, (what, msg)
    assert call(p=3, hist=(h1, h2, None)) != 0 and "history slot 3" in lib.tng_last_error().decode()
