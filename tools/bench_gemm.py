"""Micro-benchmark of tng_conv_gemm shapes (CUDA-graph replays, so no host overhead in the timing).

Besides TFLOP/s and algorithmic HBM GB/s, each line gives the L2 -> SM operand rate the plan implies: every work item
loads (bm + bn) x 64 bf16 per K block into the shared-memory ring, so the bytes drawn from L2 are
M tiles x N tiles x K blocks x (bm + bn) x 128 (split-K splits the K blocks of a tile, not the total)."""
import os, sys, math
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tango_b200 import lib as L, ops

dev = torch.device("cuda:0")

def plan(fn):
    """(block_n, M tile, ksplit) of the one tng_conv_gemm launch fn makes, from the profiler's instantiation label."""
    L.PROF.start()
    try:
        fn()
    finally:
        fam = next(iter(L.PROF.stop()))
    bn = int(fam[len("gemm_tc<"):].split(",")[0].rstrip(">"))
    return bn, 256 if ",m256" in fam else 128, 2 if ",splitk" in fam else 1


def m_tiles(NB, H, W, bm):
    """M tiles of plan_gemm's box rule: bw x bh x bn output pixels with product bm."""
    if W >= bm or H == 1:
        return NB * H * -(-W // bm)
    rem = bm // W
    return NB * -(-H // rem) if H >= rem else -(-NB // (rem // H))


def bench(name, fn, flops, bytes_, grid, N, kblocks, reps=20):
    bn, bm, ks = plan(fn)
    l2 = m_tiles(*grid, bm) * -(-N // bn) * kblocks * (bm + bn) * 128
    fn(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    tile = f"{bm}x{bn}" + (" split-K" if ks > 1 else "")
    print(f"{name:58s} {tile:15s} {us:8.1f} us  {flops/us/1e6:8.1f} TF/s  {bytes_/us/1e3:8.1f} GB/s  "
          f"{l2/us/1e3:8.1f} L2->SM GB/s")

def linear_case(M, N, K, res=True, f32=True, bf=False, bn=0, geglu=0):
    w = torch.randn(N, K, device=dev) / math.sqrt(K)
    pc = ops.PackedConv(w, torch.zeros(N, device=dev), split=False, device=dev, geglu_bn=geglu)
    x = torch.randn(M, K, device=dev).to(torch.bfloat16)
    No = N // 2 if geglu else N
    r = torch.randn(M, No, device=dev) if res else None
    of = torch.empty(M, No, device=dev) if f32 else None
    ob = torch.empty(M, No, device=dev, dtype=torch.bfloat16) if bf else None
    by = M * K * 2 + N * K * 2 + (M * No * 4 if res else 0) + (M * No * 4 if f32 else 0) + (M * No * 2 if bf else 0)
    bench(f"linear M={M} N={N} K={K} res={int(res)} f32={int(f32)} bf16={int(bf)} bn={bn} geglu={geglu}",
          lambda: ops.run_linear(pc, x, res=r, out_f32=of, out_bf16=ob, block_n=bn), 2.0 * M * N * K, by,
          (1, 1, M), N, sum(g[5] for g in pc.groups()))

def conv_case(NB, H, W, Cin, Cout, res=True):
    w = torch.randn(Cout, Cin, 3, 3, device=dev) / math.sqrt(9 * Cin)
    pc = ops.PackedConv(w, torch.zeros(Cout, device=dev), split=False, device=dev)
    x = torch.randn(NB * H * W, Cin, device=dev).to(torch.bfloat16)
    r = torch.randn(NB * H * W, Cout, device=dev) if res else None
    of = torch.empty(NB * H * W, Cout, device=dev)
    M = NB * H * W
    by = M * Cin * 2 + Cout * Cin * 18 + M * Cout * 4 * (2 if res else 1)
    bench(f"conv3x3 {NB}x{H}x{W} Cin={Cin} Cout={Cout} res={int(res)}", lambda: ops.run_conv(pc, x, NB, H, W, res=r, out_f32=of),
          2.0 * M * Cout * Cin * 9, by, (NB, H, W), Cout, sum(g[5] for g in pc.groups()))

linear_case(65536, 320, 320)
linear_case(65536, 320, 320, res=False)
linear_case(65536, 320, 320, res=False, f32=False, bf=True)
linear_case(65536, 960, 320, res=False, f32=False, bf=True)
linear_case(65536, 2560, 320, res=False, f32=False, bf=True, geglu=256)
linear_case(65536, 320, 1280, res=True)
linear_case(16384, 640, 640)
linear_case(16384, 1920, 640, res=False, f32=False, bf=True)
linear_case(16384, 5120, 640, res=False, f32=False, bf=True, geglu=256)
linear_case(4096, 1280, 1280)
linear_case(4096, 10240, 1280, res=False, f32=False, bf=True, geglu=256)
# the same problem at three N tiles: only the operand bytes per FLOP change (64.0 : 71.1 : 85.3 FLOP/B at 128 rows)
linear_case(65536, 1280, 1280, res=False, f32=False, bf=True, bn=128)
linear_case(65536, 1280, 1280, res=False, f32=False, bf=True, bn=160)
linear_case(65536, 1280, 1280, res=False, f32=False, bf=True, bn=256)
linear_case(8192, 8192, 8192, res=False, f32=False, bf=True, bn=256)
linear_case(8192, 8192, 8192, res=False, f32=False, bf=True, bn=160)
linear_case(8192, 8192, 8192, res=False, f32=False, bf=True, bn=128)
conv_case(16, 256, 16, 320, 320)
conv_case(16, 256, 16, 640, 320)
conv_case(16, 128, 8, 640, 640)
conv_case(16, 128, 8, 1280, 640)
conv_case(16, 64, 4, 1280, 1280)
conv_case(16, 64, 4, 2560, 1280)
conv_case(16, 32, 2, 1280, 1280)
conv_case(16, 32, 2, 2560, 1280)
