"""CPU: the package's host orchestration (weight packing, persistent buffers, operator sequencing, K/V caching, CFG
shared prefix) run end to end with every kernel wrapper replaced by its executable contract (tests/cabi_spec.py), and
compared with the goldens generated from the reference. The kernels themselves are checked on the GPU
(test_kernels_gpu.py); this file makes the *Python side* of the product testable without one. Nothing here is a CPU
fallback of the product: the substitution exists only under pytest's monkeypatch."""
import os

import numpy as np
import pytest
import torch

import cabi_spec
from tango_b200 import lib as L
from tango_b200 import synth
from tango_b200.t5 import T5EncoderModel
from tango_b200.unet import UNet2DConditionModel

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CPU = torch.device("cpu")


@pytest.fixture(autouse=True)
def _spec_backend(monkeypatch):
    cabi_spec.install_spec_backend(monkeypatch)


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.mark.parametrize("precision,tol", [("split", 1e-4), ("bf16", 3e-2)])
def test_tiny_unet_orchestration_vs_reference_golden(precision, tol):
    gd = np.load(os.path.join(GOLD, "tiny_unet.npz"))
    cfg = synth.TINY_UNET_CONFIG
    u = UNet2DConditionModel.from_config(cfg, precision=precision).to(CPU)
    u.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    out = u(torch.from_numpy(gd["sample"]), torch.tensor(int(gd["t"])), torch.from_numpy(gd["ehs"]),
            encoder_attention_mask=torch.from_numpy(gd["mask"])).sample
    assert out.shape == (2, 8, 32, 16)
    assert rel(out, gd["out"]) < tol
    out2 = u(torch.from_numpy(gd["sample"]), 7, torch.from_numpy(gd["ehs"])).sample
    assert rel(out2, gd["out_nomask_t7"]) < tol


def test_cfg_shared_prefix_matches_plain_forward():
    """Under CFG both halves of the UNet batch carry the same latents: computing the pre-cross-attention prefix once
    (forward_rows(cfg_shared=True)) must give the same result as the plain forward."""
    cfg = synth.TINY_UNET_CONFIG
    u = UNet2DConditionModel.from_config(cfg, precision="split").to(CPU)
    u.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    B, H, W = 2, 32, 16
    emb, mask = synth.synth_conditioning(B, 10, cfg["cross_attention_dim"], seed=5, masked_tail=3)
    u.set_conditioning(emb, mask)
    temb = u.time_embedding_table(torch.full((2 * B,), 400.0))
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(B, 8, H, W, generator=g)
    x = u.input_rows(torch.cat([lat, lat]))
    plain = u.forward_rows(x, 2 * B, H, W, temb, temb.shape[1]).clone()
    shared = u.forward_rows(x, 2 * B, H, W, temb, temb.shape[1], cfg_shared=True)
    assert rel(shared, plain) < 1e-6


@pytest.mark.parametrize("precision,tol", [("split", 1e-4), ("bf16", 2e-2)])
def test_tiny_t5_orchestration_vs_transformers_golden(precision, tol):
    gd = np.load(os.path.join(GOLD, "tiny_t5.npz"))
    cfg = synth.TINY_T5_CONFIG
    m = T5EncoderModel.from_config(cfg, precision=precision).to(CPU)
    m.load_state_dict(synth.synth_state_dict(synth.t5_encoder_param_shapes(cfg), seed=0))
    for tag in ("", "_long"):
        out = m(torch.from_numpy(gd["ids" + tag]), torch.from_numpy(gd["mask" + tag]))[0]
        assert rel(out, gd["out" + tag]) < tol


@pytest.mark.parametrize("precision", ["split", "bf16"])
def test_vae_decoder_and_vocoder_orchestration_vs_reference_golden(precision):
    from tango_b200.vae import AutoencoderKL
    gd = np.load(os.path.join(GOLD, "tiny_vae_vocoder.npz"))
    vae = AutoencoderKL(**synth.VAE_CONFIG, precision=precision).to(CPU)
    vae.load_state_dict(synth.synth_state_dict(synth.vae_decoder_param_shapes(), seed=0))
    mel = vae.decode_first_stage(torch.from_numpy(gd["z"]))
    assert mel.shape == (1, 1, 32, 64)
    assert rel(mel, gd["mel"]) < (1e-4 if precision == "split" else 3e-2)
    wav_i16 = vae.decode_to_waveform(mel)
    assert wav_i16.dtype == np.int16 and wav_i16.shape == gd["wave_i16"].shape
    wf = vae._bufs.get("hwave_f", (1, wav_i16.shape[1]), torch.float32)
    assert rel(wf, gd["wave"]) < (2e-3 if precision == "split" else 8e-2)
    if precision == "split":
        assert np.abs(wav_i16.astype(np.int32) - gd["wave_i16"].astype(np.int32)).max() <= 40


def test_scheduler_step_orchestration_bit_exact():
    """DDPM / DDIM `step` through the coefficient-table path (what tng_sched_step consumes) reproduces the reference's
    10-step loops bit for bit (tests/golden/schedulers.npz)."""
    from tango_b200.schedulers import DDIMScheduler, DDPMScheduler
    gd = np.load(os.path.join(GOLD, "schedulers.npz"))
    x0, noises = torch.from_numpy(gd["x0"]), torch.from_numpy(gd["noises"])
    for pred in ("v_prediction", "epsilon"):
        s = DDPMScheduler.from_pretrained(prediction_type=pred)
        s.set_timesteps(10)
        x = x0.clone()
        for i, t in enumerate(s.timesteps.tolist()):
            x = s.step(torch.sin(x * 3.0 + float(t) / 1000), t, x, variance_noise=noises[i]).prev_sample
        assert np.array_equal(x.numpy(), gd[f"ddpm_loop_{pred}"])
        si = DDIMScheduler.from_pretrained(prediction_type=pred)
        si.set_timesteps(10)
        x = x0.clone()
        for t in si.timesteps.tolist():
            x = si.step(torch.sin(x * 3.0 + float(t) / 1000), t, x).prev_sample
        assert np.array_equal(x.numpy(), gd[f"ddim_loop_{pred}"])


@pytest.mark.parametrize("precision,tol", [("split", 1e-4), ("bf16", 3e-2)])
def test_vae_encoder_orchestration_vs_reference_golden(precision, tol):
    """encode_first_stage (the "next" row 2): posterior mean / std against the reference AutoencoderKL
    (tests/golden/tiny_vae_encoder.npz)."""
    from tango_b200.vae import AutoencoderKL
    gd = np.load(os.path.join(GOLD, "tiny_vae_encoder.npz"))
    vae = AutoencoderKL(**synth.VAE_CONFIG, precision=precision).to(CPU)
    sd = synth.synth_state_dict(synth.vae_decoder_param_shapes(), seed=0)
    sd.update(synth.synth_state_dict(synth.vae_encoder_param_shapes(), seed=0))
    vae.load_state_dict(sd)
    post = vae.encode_first_stage(torch.from_numpy(gd["mel"]))
    assert post.mean.shape == (2, 8, 16, 16)
    assert rel(post.mean, gd["mean"]) < tol and rel(post.std, gd["std"]) < tol
    assert torch.equal(post.mode(), post.mean)
    torch.manual_seed(3)
    z = post.sample()
    torch.manual_seed(3)
    assert torch.equal(z, post.mean + post.std * torch.randn(post.mean.shape))
    # without encoder weights the decoder still loads and encode refuses loudly
    dec_only = AutoencoderKL(**synth.VAE_CONFIG, precision=precision).to(CPU)
    dec_only.load_state_dict(synth.synth_state_dict(synth.vae_decoder_param_shapes(), seed=0))
    with pytest.raises(L.TangoB200Error):
        dec_only.encode_first_stage(torch.from_numpy(gd["mel"]))


@pytest.mark.parametrize("precision,tol", [("split", 1e-4), ("bf16", 3e-2)])
def test_mustango_unet_orchestration_vs_reference_golden(precision, tol):
    """The Mustango UNet variant (beat + chord cross-attention streams; the "next" row 4) against the fork's
    UNet2DConditionModelMusic output (tests/golden/tiny_unet_music.npz)."""
    gd = np.load(os.path.join(GOLD, "tiny_unet_music.npz"))
    cfg = synth.TINY_MUSIC_UNET_CONFIG
    u = UNet2DConditionModel.from_config(cfg, precision=precision).to(CPU)
    u.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    tt = lambda n: torch.from_numpy(gd[n])
    out = u(tt("sample"), torch.tensor(int(gd["t"])), tt("ehs"), encoder_attention_mask=tt("mask"),
            beat_features=tt("beat"), chord_features=tt("chord"), beat_attention_mask=tt("bmask"),
            chord_attention_mask=tt("cmask")).sample
    assert rel(out, gd["out"]) < tol
    with pytest.raises(L.TangoB200Error):          # the Music blocks need their two extra streams
        u(tt("sample"), 3, tt("ehs"))
    plain = UNet2DConditionModel.from_config(synth.TINY_UNET_CONFIG, precision=precision).to(CPU)
    plain.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(synth.TINY_UNET_CONFIG), seed=0))
    with pytest.raises(L.TangoB200Error):          # and Tango's blocks take none
        plain(tt("sample"), 3, tt("ehs"), beat_features=tt("beat"), chord_features=tt("chord"))


class _NoEvent:
    def __init__(self, *a, **k):
        pass

    def record(self, *a, **k):
        pass

    def elapsed_time(self, other):
        return 0.0


@pytest.mark.parametrize("precision,tol", [("split", 1e-4), ("bf16", 6e-2)])
def test_inference_loop_orchestration_vs_reference_golden(monkeypatch, precision, tol):
    """AudioDiffusion.inference (CFG duplication, per-step time-embedding rows, fused CFG + scheduler step, per-step
    noise) against the latents of the reference's own loop (tests/golden/tiny_inference.npz); eager path (CUDA-graph
    capture is a GPU-only facility and replays exactly these launches)."""
    from tango_b200.pipeline import AudioDiffusion
    from tango_b200.schedulers import DDPMScheduler
    monkeypatch.setattr(torch.cuda, "Event", _NoEvent)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    gd = np.load(os.path.join(GOLD, "tiny_inference.npz"))
    cfg = synth.TINY_UNET_CONFIG
    m = AudioDiffusion(unet_config=cfg, precision=precision, use_cuda_graph=False).to(CPU)
    m.unet.load_state_dict(synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0))
    trace = []
    lat = m.inference(["synthetic prompt"], DDPMScheduler.from_pretrained(), 4, 3.0,
                      prompt_embeds=torch.from_numpy(gd["embeds"]), boolean_prompt_mask=torch.from_numpy(gd["mask"]),
                      latents=torch.from_numpy(gd["lat0"]), noises=[torch.from_numpy(n) for n in gd["noises"]],
                      latent_shape=(32, 16), trace=trace)
    assert len(trace) == 4 and lat.shape == gd["latents"].shape
    assert rel(lat, gd["latents"]) < tol


def test_mustango_inference_loop_vs_oracle(monkeypatch):
    """MusicAudioDiffusion.inference (mustango/models.py:540-600) = the Tango loop with encoded beats / chords handed to
    the Music UNet at every step; checked against the oracle loop (its UNet is pinned to the fork's Music UNet, its loop
    to the reference's Tango loop)."""
    from oracle import pipeline as opipe
    from oracle import schedulers as osched
    from tango_b200.pipeline import AudioDiffusion
    from tango_b200.schedulers import DDPMScheduler
    monkeypatch.setattr(torch.cuda, "Event", _NoEvent)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    cfg = synth.TINY_MUSIC_UNET_CONFIG
    sd = synth.synth_state_dict(synth.unet_param_shapes(cfg), seed=0)
    B, steps, guidance, D = 1, 3, 3.0, cfg["cross_attention_dim"]
    embeds, mask = synth.synth_conditioning(B, 9, D, seed=5, masked_tail=2)
    g = torch.Generator().manual_seed(31)
    beats, chords = torch.randn(2 * B, 6, D, generator=g), torch.randn(2 * B, 4, D, generator=g)
    bmask = torch.ones(2 * B, 6, dtype=torch.bool)
    bmask[0, 1:] = False
    streams = ((beats, bmask), (chords, None))
    lat0, noises = synth.synth_noise(B, steps, shape=(8, 32, 16), seed=7)
    want = opipe.inference(sd, cfg, osched.OracleDDPM(**osched.SD21_CONFIG), embeds, mask, steps, guidance, lat0, noises,
                           extra_streams=streams)
    m = AudioDiffusion(unet_config=cfg, precision="split", use_cuda_graph=False).to(CPU)
    m.unet.load_state_dict(sd)
    lat = m.inference(["x"], DDPMScheduler.from_pretrained(), steps, guidance, prompt_embeds=embeds,
                      boolean_prompt_mask=mask, latents=lat0, noises=noises, latent_shape=(32, 16), extra_streams=streams)
    assert rel(lat, want) < 1e-4


def test_tango_generate_prompt_to_waveform_vs_oracle(monkeypatch):
    """Tango.generate / generate_for_batch (tango.py:43-64) end to end on the tiny architecture: prompt -> synthetic text
    states -> CFG loop -> VAE decoder -> HiFi-GAN -> int16, against the oracle pipeline on the same conditioning and
    noise. Also the DDIM / no-CFG branch (models.py:214,218-221)."""
    from oracle import hifigan as ohifi
    from oracle import pipeline as opipe
    from oracle import schedulers as osched
    from oracle import vae as ovae
    from tango_b200.pipeline import Tango
    monkeypatch.setattr(torch.cuda, "Event", _NoEvent)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    cfg = synth.TINY_UNET_CONFIG
    t = Tango.from_synthetic(unet_config=cfg, device="cpu", precision="split")
    t.model.use_cuda_graph = False
    prompts = ["a dog barking in the rain", "church bells"]
    lat0, noises = synth.synth_noise(2, 3, shape=(8, 32, 16), seed=11)
    waves = t.generate_for_batch(prompts, steps=3, guidance=3, batch_size=2, latent_shape=(32, 16), latents=lat0,
                                 noises=noises)
    assert len(waves) == 2 and all(w.dtype == np.int16 and w.shape == (20512,) for w in waves)
    # the oracle on the same conditioning
    pe, pm = t.model.encode_text_classifier_free(prompts, 1)
    usd = synth.synth_state_dict(synth.unet_param_shapes(cfg), 0)
    vsd = synth.synth_state_dict(synth.vae_decoder_param_shapes(), 0)
    lat = opipe.inference(usd, cfg, osched.OracleDDPM(**osched.SD21_CONFIG), pe, pm, 3, 3.0, lat0, noises)
    mel = ovae.decode_first_stage(vsd, lat, synth.VAE_CONFIG["scale_factor"])
    wref, wi_ref = ohifi.decode_to_waveform(vsd, mel)
    got = np.stack(waves).astype(np.int32)
    assert np.abs(got - wi_ref.astype(np.int32)).max() <= 64            # ~2e-3 of full scale through loop + decode
    one = t.generate(prompts[0], steps=2, guidance=3, latent_shape=(32, 16))
    assert one.dtype == np.int16 and one.shape == (20512,)
    # DDIM, guidance <= 1: no CFG duplication
    from tango_b200.schedulers import DDIMScheduler
    pe1, pm1 = t.model.encode_text(prompts)
    l1 = t.model.inference(prompts, DDIMScheduler.from_pretrained(None), 3, 1.0, prompt_embeds=pe1,
                           boolean_prompt_mask=pm1, latents=lat0, latent_shape=(32, 16))
    w1 = opipe.inference(usd, cfg, osched.OracleDDIM(**osched.SD21_CONFIG), pe1, pm1, 3, 1.0, lat0)
    assert rel(l1, w1) < 1e-4


def test_tacotron_stft_orchestration_vs_reference_golden():
    """tango_b200.stft.TacotronSTFT / wav_to_fbank (the overlapping-view basis GEMM, magnitude, mel GEMM, log) against the
    reference front-end golden (tests/golden/tiny_stft.npz)."""
    from tango_b200 import stft as pstft
    gd = np.load(os.path.join(GOLD, "tiny_stft.npz"))
    FL, HOP, WIN, NMEL, target = (int(v) for v in gd["cfg"])
    fn = pstft.TacotronSTFT(FL, HOP, WIN, NMEL, 16000, 0, 8000).to(CPU)
    assert fn.mel_basis.shape == (NMEL, FL // 2 + 1) and fn.mel_basis_source.startswith("slaney")
    r = fn.load_state_dict({"mel_basis": torch.from_numpy(gd["mel_basis"])}, strict=False)
    assert "stft_fn.forward_basis" in r.missing_keys and fn.mel_basis_source == "checkpoint"
    with pytest.raises(RuntimeError):
        fn.load_state_dict({"mel_basis": torch.zeros(3, 3)}, strict=False)
    fbank, log_mag, wav = pstft.wav_to_fbank([torch.from_numpy(gd["wave0"]), torch.from_numpy(gd["wave1"])],
                                             target_length=target, fn_STFT=fn)
    assert fbank.shape == gd["fbank"].shape and log_mag.shape == gd["log_mag"].shape
    assert torch.equal(wav, torch.from_numpy(gd["wav"]))
    e_f, e_l = rel(fbank, gd["fbank"]), rel(log_mag, gd["log_mag"])
    print(f"TacotronSTFT orchestration: fbank rel {e_f:.3e}, log-mag rel {e_l:.3e}")
    assert e_f < 1e-4 and e_l < 1e-4
    with pytest.raises(AssertionError):
        fn.mel_spectrogram(torch.full((1, 4000), 1.5))


def test_slaney_mel_basis_known_properties():
    """The default mel filter bank (used only when no checkpoint is loaded): triangles on the Slaney scale, area-normalised."""
    from tango_b200.stft import slaney_mel_basis
    mb = slaney_mel_basis(16000, 1024, 64, 0, 8000)
    assert mb.shape == (64, 513) and float(mb.min()) >= 0
    peaks = mb.argmax(1)
    assert bool((peaks[1:] > peaks[:-1]).all())                      # centre frequencies increase
    # below 1 kHz the scale is linear: equal widths, equal heights
    assert abs(float(mb[2].max() / mb[3].max()) - 1.0) < 0.2
    assert float(mb[:, 0].sum()) == 0.0 or float(mb[0, 0]) == 0.0   # DC bin carries no weight at fmin = 0
