"""CPU: host-side logic of the product (no GPU compute): scheduler grids / coefficient tables against the oracle,
weight packing, state_dict shapes, k-group construction, and that GPU-only entry points refuse CPU tensors."""
import os

import numpy as np
import pytest
import torch

import cabi_spec
from oracle import schedulers as osched
from tango_b200 import ops, synth
from tango_b200 import schedulers as S


def spec_step(coef, v, s, noise):
    """tng_sched_step (latent_step.cu, SchedStep) without CFG on NCHW tensors, through cabi_spec.spec_sched_step."""
    B, Cc = s.shape[:2]
    HW = s[0, 0].numel()
    prev = torch.empty(s.shape)
    cabi_spec.spec_sched_step(v.reshape(B, Cc, HW).transpose(1, 2).reshape(B * HW, Cc), False, 1.0, s, noise, coef,
                              prev, None, B=B, Cc=Cc, HW=HW)
    return prev


@pytest.mark.parametrize("n", [10, 100, 200])
def test_timestep_grids_match_oracle(n):
    d, o = S.DDPMScheduler.from_pretrained(), osched.OracleDDPM(**osched.SD21_CONFIG)
    d.set_timesteps(n)
    o.set_timesteps(n)
    assert d.timesteps.dtype == torch.int64 and torch.equal(d.timesteps, o.timesteps)
    di, oi = S.DDIMScheduler.from_pretrained(), osched.OracleDDIM(**osched.SD21_CONFIG)
    di.set_timesteps(n)
    oi.set_timesteps(n)
    assert torch.equal(di.timesteps, oi.timesteps)
    assert d.init_noise_sigma == 1.0 and d.order == 1
    with pytest.raises(ValueError):
        d.set_timesteps(1001)


@pytest.mark.parametrize("pred", ["v_prediction", "epsilon"])
def test_coefficient_tables_bit_exact_vs_oracle(pred):
    g = torch.Generator().manual_seed(0)
    s0 = torch.randn(2, 8, 16, 16, generator=g)
    cfg = dict(osched.SD21_CONFIG, prediction_type=pred)
    for n in (10, 200):
        d = S.DDPMScheduler.from_pretrained(prediction_type=pred)
        d.set_timesteps(n)
        o = osched.OracleDDPM(**cfg)
        o.set_timesteps(n)
        tab = d.coefficient_table()
        assert tab.shape == (n, S.NCOEF) and tab.dtype == torch.float32
        x = s0.clone()
        for i, t in enumerate(o.timesteps[:12]):
            v = torch.sin(x * 2 + i)
            nz = torch.randn(x.shape, generator=g)
            ref = o.step(v, t, x, nz if int(t) > 0 else None)
            got = spec_step(tab[i], v, x, nz)
            assert torch.equal(ref, got)
            x = ref
        # last step (t == 0): no noise
        t = o.timesteps[-1]
        assert torch.equal(o.step(x, t, x), spec_step(tab[-1], x, x, None))
        di = S.DDIMScheduler.from_pretrained(prediction_type=pred)
        di.set_timesteps(n)
        oi = osched.OracleDDIM(**cfg)
        oi.set_timesteps(n)
        tabi = di.coefficient_table()
        x = s0.clone()
        for i, t in enumerate(oi.timesteps[:12]):
            v = torch.cos(x * 2 + i)
            ref = oi.step(v, t, x)
            assert torch.equal(ref, spec_step(tabi[i], v, x, None))
            x = ref


def test_off_grid_step_keeps_the_grid_table(monkeypatch):
    """DDPM / DDIM `step` at a timestep outside the grid computes that timestep's row on its own: the grid's
    coefficient_table() is unchanged, and a later step on the grid still takes its table row."""
    cabi_spec.install_spec_backend(monkeypatch)     # `step` refuses CPU tensors
    g = torch.Generator().manual_seed(3)
    x, v, nz = (torch.randn(2, 8, 4, 4, generator=g) for _ in range(3))
    for s in (S.DDPMScheduler.from_pretrained(), S.DDIMScheduler.from_pretrained()):
        s.set_timesteps(10)
        full = s.coefficient_table().clone()
        assert 7 not in s.timesteps.tolist()
        got = s.step(v, 7, x, variance_noise=nz).prev_sample
        assert torch.equal(got, spec_step(s._coefficients(7), v, x, nz if s._needs_noise(7) else None))
        assert s.coefficient_table().shape == (10, S.NCOEF) and torch.equal(s.coefficient_table(), full)
        t = int(s.timesteps[3])
        got = s.step(v, t, x, variance_noise=nz).prev_sample
        assert torch.equal(got, spec_step(full[3], v, x, nz if s._needs_noise(t) else None))


def test_unet_shapes_and_param_count():
    sh = synth.unet_param_shapes(synth.BASE_UNET_CONFIG)
    assert len(sh) == 686
    assert sum(int(np.prod(v)) for v in sh.values()) == 865_933_768
    shx = synth.unet_param_shapes(synth.XL_UNET_CONFIG)
    assert sum(int(np.prod(v)) for v in shx.values()) == 891_492_808
    assert sh["down_blocks.0.attentions.0.transformer_blocks.0.attn2.to_k.weight"] == (320, 1024)
    assert sh["up_blocks.1.resnets.0.conv_shortcut.weight"] == (1280, 2560, 1, 1)
    assert len(synth.vae_decoder_param_shapes()) == 308


def test_packed_conv_layout_and_groups():
    w = torch.arange(4 * 8 * 9, dtype=torch.float32).reshape(4, 8, 3, 3) / 100
    pc = ops.PackedConv(w, torch.zeros(4), split=False, device="cpu")
    assert pc.weight.shape == (4, 72) and pc.weight.dtype == torch.bfloat16
    # K index = tap * Cin + cin, tap = ky * 3 + kx
    assert torch.equal(pc.weight[:, 3 * 8 + 2].float(), w[:, 2, 1, 0].to(torch.bfloat16).float())
    g = pc.groups()
    assert len(g) == 9 and g[0] == (0, 0, -1, -1, 0, 1) and g[8] == (0, 0, 1, 1, 64, 1)
    pcs = ops.PackedConv(w, None, split=True, device="cpu")
    assert pcs.weight.shape == (4, 144)
    hi, lo = pcs.weight[:, :72].float(), pcs.weight[:, 72:].float()
    assert (hi + lo - w.permute(0, 2, 3, 1).reshape(4, 72)).abs().max() < 5e-5
    gs = pcs.groups(lo_views=[1])
    assert len(gs) == 27 and gs[1][0] == 1 and gs[2][4] == 72
    # stride 2: parity plane and plane offset per tap
    w2 = torch.randn(64, 64, 3, 3)
    p2 = ops.PackedConv(w2, None, split=False, device="cpu", stride=2)
    g2 = p2.groups(parity_views=[0, 1, 2, 3])
    assert g2[0][:4] == (3, 0, -1, -1) and g2[4][:4] == (0, 0, 0, 0) and g2[5][:4] == (1, 0, 0, 0)
    # GEGLU interleave
    wl = torch.arange(16 * 4, dtype=torch.float32).reshape(16, 4)
    pg = ops.PackedConv(wl, torch.arange(16, dtype=torch.float32), split=False, device="cpu", geglu_bn=8)
    assert pg.bias.tolist() == [0, 1, 2, 3, 8, 9, 10, 11, 4, 5, 6, 7, 12, 13, 14, 15]


def test_no_cpu_fallback():
    from tango_b200 import lib as L
    x = torch.zeros(4, 8)
    with pytest.raises(L.TangoB200Error):
        L.layernorm(x, torch.ones(8), torch.zeros(8), 1e-5, torch.zeros(4, 8, dtype=torch.bfloat16))
    d = S.DDPMScheduler.from_pretrained()
    d.set_timesteps(10)
    with pytest.raises(L.TangoB200Error):
        d.step(torch.zeros(1, 8, 4, 4), 990, torch.zeros(1, 8, 4, 4))


def test_t5_relative_bucket_table_matches_oracle():
    from oracle import t5 as ot5
    from tango_b200.t5 import relative_position_buckets
    for Lt in (1, 2, 10, 64, 150, 512):
        pos = torch.arange(Lt)
        want = ot5.relative_position_bucket(pos[None, :] - pos[:, None], 32, 128)      # [query, key]
        tab = relative_position_buckets(Lt, 32, 128)                                     # index key - query + L - 1
        got = tab[(pos[None, :] - pos[:, None]) + Lt - 1]
        assert torch.equal(got, want)


def test_t5_param_shapes_and_state_dict_contract():
    from tango_b200 import synth
    from tango_b200.t5 import T5EncoderModel
    shp = synth.t5_encoder_param_shapes(synth.FLAN_T5_LARGE_CONFIG)
    n = sum(int(torch.tensor(s).prod()) for s in shp.values())
    assert n == 341_231_104                       # google/flan-t5-large encoder + shared embedding
    m = T5EncoderModel.from_config(synth.TINY_T5_CONFIG)
    sd = synth.synth_state_dict(synth.t5_encoder_param_shapes(synth.TINY_T5_CONFIG), 0)
    sd2 = dict(sd)
    sd2["encoder.embed_tokens.weight"] = sd2.pop("shared.weight")      # checkpoints may carry only the tied copy
    assert not m.load_state_dict(sd2).missing_keys
    bad = dict(sd)
    bad.pop("encoder.final_layer_norm.weight")
    with pytest.raises(RuntimeError):
        m.load_state_dict(bad)
    with pytest.raises(Exception):                # no CPU fallback
        m(torch.zeros(1, 4, dtype=torch.long))


def test_fallback_tokenizer_padding_and_truncation():
    """The call conventions models.py:131-133 / :268-286 rely on: padding=True pads to the longest prompt,
    padding="max_length" to max_length, EOS closes every row, the empty prompt is a lone EOS."""
    from tango_b200.pipeline import FallbackTokenizer
    tok = FallbackTokenizer(100)
    b = tok(["a b c", "a"], max_length=tok.model_max_length, padding=True, truncation=True, return_tensors="pt")
    assert b.input_ids.shape == (2, 4) and b.attention_mask.tolist() == [[1, 1, 1, 1], [1, 1, 0, 0]]
    assert b.input_ids[0, 3] == 1 and b.input_ids[1, 1] == 1 and b.input_ids[1, 2] == 0
    assert int(b.input_ids[0, 0]) == int(b.input_ids[1, 0]) >= 2            # same word, same id, never pad/EOS
    u = tok([""], max_length=4, padding="max_length", truncation=True, return_tensors="pt")
    assert u.input_ids.tolist() == [[1, 0, 0, 0]] and u.attention_mask.tolist() == [[1, 0, 0, 0]]
    t = tok(["w " * 50], max_length=8, padding=True, truncation=True)
    assert t.input_ids.shape == (1, 8) and t.input_ids[0, -1] == 1


def test_t5_config_recovered_from_state_dict():
    from tango_b200 import synth
    from tango_b200.pipeline import t5_config_from_state_dict
    cfg = dict(synth.FLAN_T5_LARGE_CONFIG, num_layers=2, vocab_size=64)
    shapes = synth.t5_encoder_param_shapes(cfg)
    te = {k: torch.empty(s, device="meta") for k, s in shapes.items()}
    assert t5_config_from_state_dict(te) == cfg


def test_cli_manifest_wav_and_paths(tmp_path):
    """tango_b200.cli host pieces: inference_hf.py:30-66 argument names/defaults, :86-87 manifest parsing,
    :91-93 output directory naming, :107 16 kHz PCM-16 wav files."""
    import json
    import wave
    from tango_b200 import cli
    a = cli.parse_args([])
    assert (a.checkpoint, a.test_file, a.text_key, a.device) == ("declare-lab/tango", "data/test_audiocaps_subset.json",
                                                                 "captions", "cuda:0")
    assert (a.num_steps, a.guidance, a.batch_size) == (200, 3, 8)
    man = tmp_path / "prompts.json"
    man.write_text("\n".join(json.dumps({"captions": c, "id": i}) for i, c in enumerate(["a dog", "rain", "bells"])) + "\n\n")
    assert cli.read_prompts(str(man), "captions") == ["a dog", "rain", "bells"]
    assert cli.output_dir_for("outputs", "17", 200, 3.0) == "outputs/17_steps_200_guidance_3.0"
    x = (np.sin(np.arange(1600) / 10.0) * 20000).astype(np.int16)
    cli.write_wav(str(tmp_path / "o.wav"), x)
    with wave.open(str(tmp_path / "o.wav")) as w:
        assert (w.getnchannels(), w.getsampwidth(), w.getframerate(), w.getnframes()) == (1, 2, 16000, 1600)
        assert np.array_equal(np.frombuffer(w.readframes(1600), dtype="<i2"), x)
    with pytest.raises(TypeError):
        cli.write_wav(str(tmp_path / "f.wav"), x.astype(np.float32))


def test_cli_main_flow_with_stub_model(tmp_path, monkeypatch):
    """The whole CLI flow on the CPU with the model stubbed out: sharded indices, wav files, summary line."""
    import json
    from types import SimpleNamespace
    from tango_b200 import cli
    man = tmp_path / "p.json"
    man.write_text("\n".join(json.dumps({"captions": f"prompt {i}"}) for i in range(5)))
    calls = []

    class Stub:
        scheduler = SimpleNamespace(config={"num_train_timesteps": 1000})
        model = SimpleNamespace(text_encoder=SimpleNamespace(synthetic=True))

        def generate_for_batch(self, prompts, steps, guidance, batch_size, **kw):
            calls.append((list(prompts), steps, guidance, batch_size, kw))
            return [np.full(1600, i, dtype=np.int16) for i in range(len(prompts))]

    monkeypatch.setattr(cli, "build_tango", lambda *a, **k: Stub())
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    res = cli.main(["--test_file", str(man), "--num_steps", "7", "--guidance", "2.5", "--batch_size", "4",
                    "--output_root", str(tmp_path / "o"), "--exp_id", "x", "--latent_h", "32"])
    assert calls == [([f"prompt {i}" for i in range(5)], 7, 2.5, 4, {"shard": False, "latent_shape": (32, 16)})]
    out = tmp_path / "o" / "x_steps_7_guidance_2.5"
    assert res["output_dir"] == str(out) and sorted(os.listdir(out)) == [f"output_{j}.wav" for j in range(5)]
    assert abs(res["audio_seconds"] - 0.5) < 1e-9 and res["text_encoder"] == "synthetic"
    line = json.loads((tmp_path / "o" / "tango_checkpoint_summary.jsonl").read_text().strip())
    assert line["Steps"] == 7 and line["Test Instances"] == 5 and line["scheduler_config"] == {"num_train_timesteps": 1000}


def test_product_scheduler_tables_meet_reference_loop_constants():
    """The product's host-side coefficient tables (what tng_sched_step consumes), driven through the fork's own
    full-loop known answers: schedulers/test_scheduler_ddim.py:106-140 (172.0067 / 52.5302 / 149.8295 / 149.0784) and
    test_scheduler_ddpm.py:71-131 (258.9606 / 202.0296; 1000 steps, seeded noise)."""
    n = 4 * 3 * 8 * 8
    x_init = (torch.arange(n).reshape(3, 8, 8, 4) / n).permute(3, 0, 1, 2)       # dummy_sample_deter
    model = lambda s, t: s * t / (t + 1)                                            # dummy_model
    base = dict(num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear", clip_sample=True)
    for extra, es, em in ((dict(prediction_type="epsilon"), 172.0067, 0.223967),
                          (dict(prediction_type="v_prediction"), 52.5302, 0.0684),
                          (dict(set_alpha_to_one=True, beta_start=0.01), 149.8295, 0.1951),
                          (dict(set_alpha_to_one=False, beta_start=0.01), 149.0784, 0.1941)):
        d = S.DDIMScheduler(**dict(base, **extra))
        d.set_timesteps(10)
        tab = d.coefficient_table()
        x = x_init.clone()
        for i, t in enumerate(d.timesteps):
            x = spec_step(tab[i], model(x, t), x, None)
        assert abs(x.abs().sum().item() - es) < 1e-2 and abs(x.abs().mean().item() - em) < 1e-3
    for pred, es, em in (("epsilon", 258.9606, 0.3372), ("v_prediction", 202.0296, 0.2631)):
        d = S.DDPMScheduler(**dict(base, prediction_type=pred))
        d.set_timesteps(1000)
        tab = d.coefficient_table()
        x = x_init.clone()
        g = torch.manual_seed(0)
        for i, t in enumerate(d.timesteps):
            res = model(x, t)
            noise = torch.randn(res.shape, generator=g) if int(t) > 0 else None
            x = spec_step(tab[i], res, x, noise)
        assert abs(x.abs().sum().item() - es) < 1e-2 and abs(x.abs().mean().item() - em) < 1e-3


def test_generate_for_batch_chunking_sharding_and_generator_routing(monkeypatch):
    """Host logic of Tango.generate_for_batch (tango.py:51-64 + the shard / seed contract of SURVEY.md section 8e) with
    the model and decoder stubbed: chunks of batch_size, contiguous split of every chunk over the ranks, the row window
    handed to the noise draws, per-sample generator lists sliced per chunk and rank, empty shards advancing the RNG."""
    import numpy as np
    from tango_b200 import parallel
    from tango_b200.pipeline import Tango

    calls, advanced = [], []

    class _Model:
        use_cuda_graph = False

        def inference(self, prompts, scheduler, steps, guidance, samples, disable_progress=True, generator=None,
                      noise_rows=None, **kw):
            calls.append((list(prompts), samples, generator, noise_rows))
            return torch.zeros(len(prompts) * samples, 8, 4, 4)

        def advance_rng(self, total, scheduler, steps, generator, latent_shape):
            advanced.append((total, generator))

    t = Tango.__new__(Tango)
    t.model, t.scheduler, t.device = _Model(), object(), torch.device("cpu")
    ids = iter(range(10 ** 6))
    t._decode = lambda lat: np.stack([np.full(3, next(ids), dtype=np.int16) for _ in range(lat.shape[0])])
    prompts = [f"p{i}" for i in range(5)]

    # single process: chunks of 2, 2, 1; samples = 2 -> groups of 2 waveforms per prompt, generator passed through
    out = t.generate_for_batch(prompts, steps=1, guidance=3, samples=2, batch_size=2, generator="G")
    assert [c[0] for c in calls] == [["p0", "p1"], ["p2", "p3"], ["p4"]] and all(c[2] == "G" and c[3] is None for c in calls)
    assert len(out) == 5 and all(len(o) == 2 for o in out)
    # per-sample generator list: sliced per chunk (2 prompts x 2 samples = 4 generators per chunk)
    calls.clear()
    gens = [f"g{i}" for i in range(10)]
    t.generate_for_batch(prompts, steps=1, guidance=3, samples=2, batch_size=2, generator=gens)
    assert [c[2] for c in calls] == [gens[0:4], gens[4:8], gens[8:10]]
    with pytest.raises(ValueError):
        t.generate_for_batch(prompts, steps=1, guidance=3, samples=2, batch_size=2, generator=gens[:7])
    # world of 2, rank 1: chunk [p0..p3] -> rows 2..3 of 4; chunk [p4] -> empty shard, RNG advanced instead
    calls.clear()
    monkeypatch.setattr(parallel, "world_size", lambda: 2)
    monkeypatch.setattr(parallel, "rank", lambda: 1)
    monkeypatch.setattr(parallel, "allgather_waves", lambda w, dev=None: w)
    out = t.generate_for_batch(prompts, steps=7, guidance=3, samples=1, batch_size=4, generator="G", shard=True)
    assert calls == [(["p2", "p3"], 1, "G", (2, 4, 4))]
    assert advanced == [(1, "G")] and len(out) == 2
    # shard=False ignores the process group
    calls.clear()
    t.generate_for_batch(prompts[:2], steps=1, guidance=3, batch_size=8)
    assert calls[0][0] == ["p0", "p1"] and calls[0][3] is None
