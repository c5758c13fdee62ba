"""Time the flash-attention entry points at the shapes the Tango UNet and VAE run, next to what bounds them.

    python tools/bench_attn.py [--lib PATH] [--json PATH] [--windows N]

For every shape it prints the kernel time (median of N event-timed windows, each a CUDA graph of back-to-back
launches), the algorithmic rate (4·B·heads·Lq·Lk·D FLOP: QKᵀ plus PV) and two floors at the card's maximum SM clock:
the tensor floor (FLOP over 4096 dense bf16 FLOP/clk/SM) and the MUFU floor (one ex2 per score, padded query / key
tiles included, over 16 ex2/clk/SM, i.e. what the softmax would cost if every exponential ran on MUFU). The card's
name, power limit and SM clocks are read in the same call. --lib times another build of libtango_b200.so (for example
the parent commit's), so that two builds can be compared by alternating runs of this script.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tango_b200 import build as _build
from tango_b200 import lib as L

FA_BM, FA_BN = 128, 64          # queries per CTA, keys per tile (attention.cu)
TENSOR_FLOP_PER_CLK_SM = 4096   # dense bf16 wgmma, H100
MUFU_EX2_PER_CLK_SM = 16

# (name, B, heads, Lq, Lk): the UNet's attention at UNet batch 16 (8 prompts under CFG), 10.24 s clips (256 x 16
# latents); self-attention at the three resolutions, cross-attention over 64 text tokens
UNET_SHAPES = [
    ("self 256x16", 16, 5, 4096, 4096),
    ("self 128x8", 16, 10, 1024, 1024),
    ("self 64x4", 16, 20, 256, 256),
    ("cross 256x16", 16, 5, 4096, 64),
    ("cross 128x8", 16, 10, 1024, 64),
    ("cross 64x4", 16, 20, 256, 64),
    ("cross 32x2", 16, 20, 64, 64),
]
EXTRA_SHAPES = [("self 768x16 (30 s)", 8, 5, 12288, 12288)]
WIDE_SHAPES = [("vae 10 s", 8, 4096), ("vae 30 s", 8, 12288)]


def card_info():
    info = {"name": torch.cuda.get_device_name(0), "sms": torch.cuda.get_device_properties(0).multi_processor_count}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                              "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        pl, sm, smax = (float(v) for v in out.split(","))
        info.update(power_limit_w=pl, sm_clock_mhz=sm, max_sm_clock_mhz=smax)
    except (OSError, ValueError, subprocess.SubprocessError):
        info.update(power_limit_w=None, sm_clock_mhz=None, max_sm_clock_mhz=None)
    return info


def time_us(fn, reps, windows):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / reps)
    return statistics.median(ts)


def floors_us(flop, ex2, sms, mhz):
    if not mhz:
        return None, None
    clk = sms * mhz * 1e6
    return flop / (TENSOR_FLOP_PER_CLK_SM * clk) * 1e6, ex2 / (MUFU_EX2_PER_CLK_SM * clk) * 1e6


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", default=None, help="path of the libtango_b200.so to time (default: the in-tree build)")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    ap.add_argument("--windows", type=int, default=5, help="timed windows per shape (median reported)")
    ap.add_argument("--no-extra", action="store_true", help="only the UNet shapes at batch 16")
    args = ap.parse_args()
    if args.lib:
        _build.LIB_PATH = os.path.abspath(args.lib)
    L.load(build_if_missing=args.lib is None)
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    rows = []

    def bench(name, B, heads, Lq, Lk):
        Cc = heads * 64
        q = torch.randn(B * Lq, 3 * Cc, device=dev).to(torch.bfloat16)
        kv = q if Lk == Lq else torch.randn(B * Lk, 3 * Cc, device=dev).to(torch.bfloat16)
        out = torch.empty(B * Lq, Cc, device=dev, dtype=torch.bfloat16)
        flop = 4.0 * B * heads * Lq * Lk * 64
        reps = max(3, min(50, int(3e11 / flop)))
        us = time_us(lambda: L.attention(q, kv, kv, out, batch=B, heads=heads, Lq=Lq, Lk=Lk, scale=0.125, k_col0=Cc,
                                         v_col0=2 * Cc), reps, args.windows)
        lq_pad = -(-Lq // FA_BM) * FA_BM
        lk_pad = -(-Lk // FA_BN) * FA_BN
        ex2 = B * heads * lq_pad * (lk_pad + 2 * lk_pad // FA_BN)   # scores + the two running-max corrections / tile
        rows.append(dict(kind="attention", name=name, B=B, heads=heads, Lq=Lq, Lk=Lk, us=us, tflops=flop / us / 1e6,
                         flop=flop, ex2=ex2))

    def bench_wide(name, B, L_):   # the VAE AttnBlock: one head of width 512
        Cc = 512
        qkv = torch.randn(B * L_, 3 * Cc, device=dev).to(torch.bfloat16)
        out = torch.empty(B * L_, Cc, device=dev, dtype=torch.bfloat16)
        flop = 4.0 * B * L_ * L_ * Cc
        us = time_us(lambda: L.attention_wide(qkv, qkv, qkv, out, batch=B, L=L_, dim=Cc, scale=Cc ** -0.5,
                                              k_col0=Cc, v_col0=2 * Cc), 3, args.windows)
        rows.append(dict(kind="attention_wide", name=name, B=B, heads=1, Lq=L_, Lk=L_, us=us,
                         tflops=flop / us / 1e6, flop=flop, ex2=2 * B * L_ * L_))

    for s in UNET_SHAPES:
        bench(*s)
    if not args.no_extra:
        for s in EXTRA_SHAPES:
            bench(*s)
        for s in WIDE_SHAPES:
            bench_wide(*s)
    card = card_info()   # read right after the timed work, while the clocks are still those of the load
    for r in rows:
        r["tensor_floor_us"], r["mufu_floor_us"] = floors_us(r["flop"], r["ex2"], card["sms"], card["max_sm_clock_mhz"])
    print(f"# {card['name']}, {card['sms']} SMs, power limit {card['power_limit_w']} W, SM clock "
          f"{card['sm_clock_mhz']} MHz after the runs (max {card['max_sm_clock_mhz']}); floors at the max clock")
    print(f"# lib {L.lib_path()}")
    print(f"{'shape':<20} {'B':>3} {'heads':>5} {'Lq':>6} {'Lk':>6} {'time us':>10} {'TFLOP/s':>8} "
          f"{'tensor floor':>13} {'MUFU floor':>11}")
    for r in rows:
        tf = f"{r['tensor_floor_us']:10.1f} us" if r["tensor_floor_us"] else "   unknown"
        mf = f"{r['mufu_floor_us']:8.1f} us" if r["mufu_floor_us"] else "  unknown"
        print(f"{r['name']:<20} {r['B']:>3} {r['heads']:>5} {r['Lq']:>6} {r['Lk']:>6} {r['us']:10.1f} "
              f"{r['tflops']:8.1f} {tf:>13} {mf:>11}")
    result = {"card": card, "lib": L.lib_path(), "rows": rows}
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
