import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tango_b200 import lib as L
dev = torch.device("cuda:0")
def time_us(fn, reps):
    fn(); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps): fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps
def bench(B, heads, Lq, Lk, reps=10):
    Cc = heads * 64
    q = torch.randn(B * Lq, 3 * Cc, device=dev).to(torch.bfloat16)
    kv = q if Lk == Lq else torch.randn(B * Lk, 3 * Cc, device=dev).to(torch.bfloat16)
    out = torch.empty(B * Lq, Cc, device=dev, dtype=torch.bfloat16)
    us = time_us(lambda: L.attention(q, kv, kv, out, batch=B, heads=heads, Lq=Lq, Lk=Lk, scale=0.125, k_col0=Cc,
                                     v_col0=2 * Cc), reps)
    print(f"attn B={B} h={heads} Lq={Lq} Lk={Lk}: {us:8.1f} us  {4.0*B*heads*Lq*Lk*64/us/1e6:7.1f} TF/s")
def bench_wide(B, L_, reps=3):   # the VAE AttnBlock: one head of width 512
    Cc = 512
    qkv = torch.randn(B * L_, 3 * Cc, device=dev).to(torch.bfloat16)
    out = torch.empty(B * L_, Cc, device=dev, dtype=torch.bfloat16)
    us = time_us(lambda: L.attention_wide(qkv, qkv, qkv, out, batch=B, L=L_, dim=Cc, scale=Cc ** -0.5, k_col0=Cc,
                                          v_col0=2 * Cc), reps)
    print(f"attn_wide B={B} d={Cc} L={L_}: {us:8.1f} us  {4.0*B*L_*L_*Cc/us/1e6:7.1f} TF/s")
bench(16, 5, 4096, 4096); bench(16, 10, 1024, 1024); bench(16, 20, 256, 256); bench(16, 5, 4096, 64); bench(16, 10, 1024, 64); bench(16, 20, 64, 64); bench(8, 5, 12288, 12288, reps=3)
bench_wide(8, 4096, reps=10); bench_wide(8, 12288)
