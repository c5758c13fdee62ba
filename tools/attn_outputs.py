"""Compare the flash-attention outputs of two builds of libtango_b200.so on the same seeded inputs.

    python tools/attn_outputs.py dump --lib A/libtango_b200.so --out a.npz
    python tools/attn_outputs.py dump --lib B/libtango_b200.so --out b.npz
    python tools/attn_outputs.py compare a.npz b.npz

`dump` runs tng_attention in both precisions (bf16, and the split mode with hi/lo operands and a hi/lo output) at the
UNet's attention shapes (UNet batch 16; self-attention at the three resolutions, masked cross-attention over 64 and
over a ragged 77 text tokens) and tng_attention_wide at the VAE shapes, and stores the raw bf16 bits. `compare` reports
for every case whether the two builds agree bit for bit and, where not, the relative L2 distance and largest absolute
difference of the hi outputs. A change that keeps the split mode and the VAE arithmetic must show them bit-identical.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

# (name, B, heads, Lq, Lk, masked)
UNET_CASES = [
    ("self 256x16", 16, 5, 4096, 4096, False),
    ("self 128x8", 16, 10, 1024, 1024, False),
    ("self 64x4", 16, 20, 256, 256, False),
    ("cross 256x16", 16, 5, 4096, 64, True),
    ("cross 128x8 Lk=77", 16, 10, 1024, 77, True),
]
VAE_CASES = [("vae 10 s", 8, 4096), ("vae 30 s", 1, 12288)]


def dump(args):
    import torch

    from tango_b200 import build as _build
    from tango_b200 import lib as L
    if args.lib:
        _build.LIB_PATH = os.path.abspath(args.lib)
    L.load(build_if_missing=args.lib is None)
    dev = torch.device("cuda:0")
    res = {}

    def rnd(gen, *shape):
        return torch.randn(*shape, generator=gen).to(dev)

    for i, (name, B, heads, Lq, Lk, masked) in enumerate(UNET_CASES):
        gen = torch.Generator().manual_seed(1000 + i)
        C = heads * 64
        q32, k32, v32 = rnd(gen, B * Lq, C), rnd(gen, B * Lk, C), rnd(gen, B * Lk, C)
        kbias = None
        if masked:   # the UNet's text mask: the last few tokens of every other prompt masked with -10000
            kb = torch.zeros(B, Lk)
            kb[1::2, Lk - 5:] = -10000.0
            kbias = kb.to(dev)

        def split(x):   # [hi | lo] as the split precision stores an operand
            hi = x.to(torch.bfloat16)
            return torch.cat([hi, (x - hi.float()).to(torch.bfloat16)], 1).contiguous()
        out = torch.zeros(B * Lq, C, device=dev, dtype=torch.bfloat16)
        L.attention(q32.to(torch.bfloat16), k32.to(torch.bfloat16), v32.to(torch.bfloat16), out, batch=B, heads=heads,
                    Lq=Lq, Lk=Lk, scale=0.125, kbias=kbias)
        res[f"bf16 | {name}"] = out.view(torch.int16).cpu().numpy()
        q2, k2, v2 = split(q32), split(k32), split(v32)
        out2 = torch.zeros(B * Lq, 2 * C, device=dev, dtype=torch.bfloat16)
        L.attention(q2, k2, v2, out2, batch=B, heads=heads, Lq=Lq, Lk=Lk, scale=0.125, kbias=kbias, nsplit=2,
                    q_lo_off=C, k_lo_off=C, v_lo_off=C, split_off=C)
        res[f"split | {name}"] = out2.view(torch.int16).cpu().numpy()
    for i, (name, B, L_) in enumerate(VAE_CASES):
        gen = torch.Generator().manual_seed(2000 + i)
        qkv = rnd(gen, B * L_, 3 * 512).to(torch.bfloat16)
        out = torch.zeros(B * L_, 512, device=dev, dtype=torch.bfloat16)
        L.attention_wide(qkv, qkv, qkv, out, batch=B, L=L_, dim=512, scale=512 ** -0.5, k_col0=512, v_col0=1024)
        res[f"wide | {name}"] = out.view(torch.int16).cpu().numpy()
    torch.cuda.synchronize()
    np.savez(args.out, **res)
    print(f"wrote {len(res)} outputs of {L.lib_path()} to {args.out}")


def bf16_bits_to_f32(a):
    return (a.astype(np.int32) << 16).view(np.float32)


def compare(args):
    a, b = np.load(args.a), np.load(args.b)
    all_split_equal = True
    for key in a.files:
        x, y = a[key], b[key]
        same = np.array_equal(x, y)
        line = f"{key:<32} {'bit-identical' if same else 'differs'}"
        if not same:
            fx, fy = bf16_bits_to_f32(x), bf16_bits_to_f32(y)
            if key.startswith("split"):   # the hi half
                fx, fy = fx[:, : fx.shape[1] // 2], fy[:, : fy.shape[1] // 2]
            d = fx.astype(np.float64) - fy
            line += (f"  rel L2 {np.linalg.norm(d) / np.linalg.norm(fx.astype(np.float64)):.3e}"
                     f"  max abs {np.abs(d).max():.3e}  differing elements {np.mean(x != y) * 100:.2f} %")
            if not key.startswith("bf16"):
                all_split_equal = False
        print(line)
    print("split mode and VAE bit-identical:", all_split_equal)
    return 0 if all_split_equal else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    sub = ap.add_subparsers(dest="cmd", required=True)
    d = sub.add_parser("dump")
    d.add_argument("--lib", default=None)
    d.add_argument("--out", required=True)
    c = sub.add_parser("compare")
    c.add_argument("a")
    c.add_argument("b")
    args = ap.parse_args()
    if args.cmd == "dump":
        dump(args)
        return 0
    return compare(args)


if __name__ == "__main__":
    sys.exit(main())
