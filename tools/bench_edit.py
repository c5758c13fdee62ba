#!/usr/bin/env python
"""Text-guided editing and inpainting on the H100: the front end, the loop with and without the per-step blend, the
decoder, whole edits, and the tng_latent_blend kernel on its own.

    python tools/bench_edit.py [--rounds 2] [--batch 8] [--kernel-iters 500] [--out FILE]

Workload: the Tango base UNet and AudioLDM VAE (seeded synthetic weights), a batch of 8 prompts (64 synthetic T5
tokens, CFG 3.0, UNet batch 16) with one 10.24 s input clip each (256 x 16 latents), bf16 precision. Reported:
  * front_end_ms: wav_to_fbank (STFT kernels) + VAE encoder for the 8 clips;
  * loop step ms of a DDPM edit (no per-step blend) and of a DDPM inpaint (one tng_latent_blend launch per step);
  * decode_ms: VAE decoder + HiFi-GAN;
  * audio-s/s of whole Tango.edit_for_batch calls (clips in, int16 out): DDPM-200 edit at strength 0.5, DPM-Solver++ 2M
    25-step edit at strength 0.6, DDPM-200 inpaint (time band 0.25-0.75) at strength 0.5;
  * tng_latent_blend alone at the loop's shapes (mask, CFG, bf16 next input): `--kernel-iters` launches replayed from
    one CUDA graph, timed with CUDA events, as us per launch and GB/s of its algorithmic bytes against 3.35 TB/s.
Every configuration is warmed up once, then the configurations alternate for `--rounds` rounds and medians are reported.
The card's name and power limit are read in the same run. One JSON line goes to stdout (and to --out). This measures
speed only: the audio quality of an edit needs pretrained weights.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.bench_dpm import card  # noqa: E402

HBM_TBPS = 3.35   # H100 SXM data sheet


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--guidance", type=float, default=3.0)
    ap.add_argument("--kernel-iters", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_edit.py: no CUDA device (the product path has no CPU fallback)")
    from tango_b200 import lib as L
    from tango_b200 import synth
    from tango_b200.pipeline import Tango, ratio_mask
    from tango_b200.schedulers import DDPMScheduler, DPMSolverMultistepScheduler
    from tango_b200.stft import wav_to_fbank
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    B, H, W, Cl = args.batch, 256, 16, 8
    audio_s = (4 * H * 160 + 32) / 16000.0
    t = Tango.from_synthetic(unet_config=synth.BASE_UNET_CONFIG, device=dev, precision="bf16")
    embeds, mask = synth.synth_conditioning(B, 64, synth.BASE_UNET_CONFIG["cross_attention_dim"], seed=1)
    embeds, mask = embeds.to(dev), mask.to(dev)
    prompts = [f"synthetic prompt {i}" for i in range(B)]
    g = torch.Generator().manual_seed(3)
    clips = [(0.3 * torch.randn(4 * H * 160, generator=g)) for _ in range(B)]
    ddpm = DDPMScheduler.from_pretrained()
    dpm = DPMSolverMultistepScheduler.from_config(ddpm.config)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, r

    def front_end():
        fb, _, _ = wav_to_fbank([c.to(dev) for c in clips], target_length=4 * H, fn_STFT=t.stft)
        return t.vae.encode_first_stage(fb.unsqueeze(1).contiguous()).mean

    x0 = t.vae.get_first_stage_encoding(front_end()).contiguous()
    band = ratio_mask(H, W, (0.25, 0.75))

    def loop(masked):
        t.model.inference(prompts, ddpm, 40, args.guidance, prompt_embeds=embeds, boolean_prompt_mask=mask,
                          latent_shape=(H, W), init_latents=x0, strength=0.5, inpaint_mask=band if masked else None,
                          generator=torch.Generator(device=dev).manual_seed(5))
        return t.model.last_step_ms

    def decode():
        rows = x0.permute(0, 2, 3, 1).reshape(B * H * W, Cl).contiguous()
        t.vae.decode_rows_to_waveform(rows, B, H, W)

    def edit(sch, steps, strength, **kw):
        t.scheduler = sch
        return t.edit_for_batch(prompts, clips, strength=strength, steps=steps, guidance=args.guidance, batch_size=B,
                                latent_shape=(H, W), prompt_embeds=embeds, boolean_prompt_mask=mask,
                                generator=torch.Generator(device=dev).manual_seed(7), **kw)

    legs = {"front_end_ms": lambda: timed(front_end)[0],
            "loop_step_ms_edit": lambda: loop(False),
            "loop_step_ms_inpaint": lambda: loop(True),
            "decode_ms": lambda: timed(decode)[0],
            "ddpm_200_edit_s0.5": lambda: timed(lambda: edit(ddpm, 200, 0.5))[0],
            "dpmsolver++2M_25_edit_s0.6": lambda: timed(lambda: edit(dpm, 25, 0.6))[0],
            "ddpm_200_inpaint_s0.5": lambda: timed(lambda: edit(ddpm, 200, 0.5,
                                                                time_mask_ratio_start_and_end=(0.25, 0.75)))[0]}
    for fn in legs.values():      # warm-up: graph capture, packed encoder, coefficient tables
        fn()
    res = {k: [] for k in legs}
    for _ in range(args.rounds):
        for k, fn in legs.items():
            res[k].append(fn())
    out = {k: float(np.median(v)) for k, v in res.items()}
    for k in ("ddpm_200_edit_s0.5", "dpmsolver++2M_25_edit_s0.6", "ddpm_200_inpaint_s0.5"):
        out[k] = {"pass_ms": out[k], "audio_s_per_s": B * audio_s / (out[k] / 1e3), "passes_ms": res[k]}
    out["blend_step_overhead_ms"] = out["loop_step_ms_inpaint"] - out["loop_step_ms_edit"]

    # ---- the kernel alone, at the loop's shapes: masked blend, CFG halves of the bf16 next input written
    HW = H * W
    gd = torch.Generator(device=dev).manual_seed(0)
    xk, nz, smp = (torch.randn(B, Cl, H, W, device=dev, generator=gd) for _ in range(3))
    mk = band.reshape(1, HW).to(dev).contiguous()
    ddpm.set_timesteps(200, device=dev)
    coef = ddpm.blend_table(dev)[100]
    x_in = torch.zeros(2 * B * HW, Cl, device=dev, dtype=torch.bfloat16)

    def launch():
        L.latent_blend(xk, nz, mk, coef, smp, x_in, B=B, Cc=Cl, HW=HW, cfg=True)

    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(args.kernel_iters):
            launch()
    graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / args.kernel_iters
    n = B * Cl * HW
    nbytes = n * 4 * 4 + HW * 4 + n * 2 * 2          # x0, noise, sample in + out; the mask; two bf16 input rows
    gbps = nbytes / (us * 1e-6) / 1e9
    kernel = {"shape": f"B={B} C={Cl} HW={HW}, one broadcast mask, CFG, bf16 next input", "launches": args.kernel_iters,
              "us_per_launch": us, "algorithmic_bytes": nbytes, "GB_per_s": gbps,
              "share_of_hbm_peak": gbps / (HBM_TBPS * 1e3),
              "timing": "CUDA events around one graph of back-to-back launches"}
    line = {"tool": "bench_edit", "card": card(), "workload": f"Tango base UNet + AudioLDM VAE, batch {B} prompts with "
            f"one {audio_s:.2f} s clip each (UNet batch {2 * B}), CFG {args.guidance}, 64 synthetic T5 tokens, bf16; "
            "loop legs: DDPM 40-step grid at strength 0.5 (20 executed steps)", "rounds": args.rounds,
            "results": out, "latent_blend_kernel": kernel}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
