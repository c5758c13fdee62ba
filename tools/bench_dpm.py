#!/usr/bin/env python
"""Few-step sampling on the H100: DDPM 200 steps against DPM-Solver++ 2M at 20 and 25 steps and UniPC-2 bh2 at 10 and
20 steps, plus the tng_dpm_step and tng_unipc_step kernels on their own.

    python tools/bench_dpm.py [--rounds 2] [--batch 8] [--kernel-iters 500] [--out FILE]

Workload: the Tango base UNet (seeded synthetic weights), a batch of 8 prompts (64 synthetic T5 tokens, CFG 3.0, UNet
batch 16), 10.24 s clips (256 x 16 latents), bf16 precision, inputs resident on the device; one pass = the denoising
loop + VAE decoder + HiFi-GAN. Every configuration is warmed up once, then the configurations are alternated for
`--rounds` rounds and the median pass is reported as audio-s/s, together with the loop's per-step time (UNet graph
replay + scheduler kernel). The kernel legs time `--kernel-iters` back-to-back tng_dpm_step launches (order 2) and
tng_unipc_step launches (order-2 corrector and predictor), at the loop's shapes and buffers, with CUDA events and divide
each kernel's algorithmic bytes by that time. The card's name
and power limit are read in the same run. One JSON line goes to stdout (and to --out).
This measures speed only: the audio quality of 20-25 DPM-Solver++ steps or 10-20 UniPC steps against 200 DDPM steps needs
pretrained weights.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [x.strip() for x in q.split(",")[:2]]
    except Exception as e:   # the numbers are still reported; the card line says why it is incomplete
        info["power_limit"] = f"unavailable ({type(e).__name__})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--guidance", type=float, default=3.0)
    ap.add_argument("--kernel-iters", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dpm.py: no CUDA device (the product path has no CPU fallback)")
    from tango_b200 import lib as L
    from tango_b200 import synth
    from tango_b200.pipeline import Tango
    from tango_b200.schedulers import DDPMScheduler, DPMSolverMultistepScheduler, UniPCMultistepScheduler
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    B, H, W = args.batch, 256, 16
    audio_s = (4 * H * 160 + 32) / 16000.0
    t = Tango.from_synthetic(unet_config=synth.BASE_UNET_CONFIG, device=dev, precision="bf16")
    embeds, mask = synth.synth_conditioning(B, 64, synth.BASE_UNET_CONFIG["cross_attention_dim"], seed=1)
    embeds, mask = embeds.to(dev), mask.to(dev)
    prompts = [f"synthetic prompt {i}" for i in range(B)]
    ddpm = DDPMScheduler.from_pretrained()
    configs = {"ddpm_200": (ddpm, 200),
               "dpmsolver++2M_20": (DPMSolverMultistepScheduler.from_config(ddpm.config), 20),
               "dpmsolver++2M_25": (DPMSolverMultistepScheduler.from_config(ddpm.config), 25),
               "unipc2_bh2_10": (UniPCMultistepScheduler.from_config(ddpm.config), 10),
               "unipc2_bh2_20": (UniPCMultistepScheduler.from_config(ddpm.config), 20)}

    def one_pass(sch, steps):
        gen = torch.Generator(device=dev).manual_seed(1234)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lat = t.model.inference(prompts, sch, steps, args.guidance, prompt_embeds=embeds, boolean_prompt_mask=mask,
                                generator=gen, latent_shape=(H, W))
        rows = lat.permute(0, 2, 3, 1).reshape(B * H * W, 8).contiguous()
        t.vae.decode_rows_to_waveform(rows, B, H, W)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, t.model.last_step_ms

    for name, (sch, steps) in configs.items():          # warm-up: graph capture, temb tables, coefficient tables
        one_pass(sch, steps)
    res = {name: {"pass_s": [], "step_ms": []} for name in configs}
    for _ in range(args.rounds):
        for name, (sch, steps) in configs.items():
            s, ms = one_pass(sch, steps)
            res[name]["pass_s"].append(s)
            res[name]["step_ms"].append(ms)
    out = {}
    for name, (sch, steps) in configs.items():
        p = float(np.median(res[name]["pass_s"]))
        out[name] = {"steps": steps, "pass_s": p, "audio_s_per_s": B * audio_s / p,
                     "loop_step_ms": float(np.median(res[name]["step_ms"])), "passes_s": res[name]["pass_s"]}
    base = out["ddpm_200"]["audio_s_per_s"]
    for name in configs:
        out[name]["speedup_vs_ddpm_200"] = out[name]["audio_s_per_s"] / base

    # ---- the kernels alone, at the loop's shapes: CFG halves in, order-2 update, bf16 next input out
    Cl, HW = 8, H * W
    n = B * Cl * HW
    g = torch.Generator(device=dev).manual_seed(0)
    model_out = torch.randn(2 * B * HW, Cl, device=dev, generator=g)
    sample = torch.randn(B, Cl, H, W, device=dev, generator=g)
    hist = [torch.randn(B, Cl, H, W, device=dev, generator=g) for _ in range(3)]
    last = torch.randn(B, Cl, H, W, device=dev, generator=g)
    x_in = torch.zeros(2 * B * HW, Cl, device=dev, dtype=torch.bfloat16)
    prev = torch.empty_like(sample)
    dpm = DPMSolverMultistepScheduler.from_config(ddpm.config)
    dpm.set_timesteps(25, device=dev)
    dpm_coef = dpm.coefficient_table(dev)[5]
    uni = UniPCMultistepScheduler.from_config(ddpm.config)
    uni.set_timesteps(10, device=dev)
    uni_coef = uni.coefficient_table(dev)[5]
    assert uni.order_at(5) == (2, 2)
    kernels = {
        "dpm_step_kernel": (lambda: L.dpm_step(model_out, True, args.guidance, sample, dpm_coef, 2, hist[0], hist[1],
                                               None, prev, x_in, B=B, Cc=Cl, HW=HW),
                            # mo halves, sample, m0, m1, prev; two bf16 input rows
                            n * 4 * (2 + 1 + 1 + 1 + 1) + n * 2 * 2, "order 2"),
        "unipc_step_kernel": (lambda: L.unipc_step(model_out, True, args.guidance, sample, uni_coef, 2, 2, hist[0],
                                                   hist[1:3], last, prev, x_in, B=B, Cc=Cl, HW=HW),
                              # mo halves, sample, m_i, m_{i-1}, m_{i-2}, last in and out, prev; two bf16 input rows
                              n * 4 * (2 + 1 + 1 + 2 + 2 + 1) + n * 2 * 2, "corrector order 2, predictor order 2")}
    kernel_out = {}
    for name, (launch, nbytes, orders) in kernels.items():
        for _ in range(20):
            launch()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()          # the same launches without the host's per-call cost between them
        with torch.cuda.graph(graph):
            for _ in range(args.kernel_iters):
                launch()
        graph.replay()
        e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
        e0.record()
        for _ in range(args.kernel_iters):
            launch()
        e1.record()
        graph.replay()
        e2.record()
        torch.cuda.synchronize()
        us_eager = e0.elapsed_time(e1) * 1e3 / args.kernel_iters
        us = e1.elapsed_time(e2) * 1e3 / args.kernel_iters
        kernel_out[name] = {"orders": orders, "shape": f"B={B} C={Cl} HW={HW}, CFG, bf16 next input",
                            "launches": args.kernel_iters, "us_per_launch": us, "algorithmic_bytes": nbytes,
                            "GB_per_s": nbytes / (us * 1e-6) / 1e9, "us_per_launch_eager": us_eager,
                            "timing": "CUDA events around a graph of back-to-back launches; _eager: the same launches "
                                      "issued one by one from Python (host bound)"}

    line = {"tool": "bench_dpm", "card": card(), "workload": f"Tango base UNet, batch {B} prompts (UNet batch {2 * B}), "
            f"CFG {args.guidance}, {audio_s:.2f} s clips, 64 synthetic T5 tokens, bf16, device-resident inputs, "
            "loop + VAE decoder + HiFi-GAN per pass", "rounds": args.rounds, "configs": out, **kernel_out}
    s = json.dumps(line)
    print(s, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
