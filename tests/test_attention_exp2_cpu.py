"""ex2_poly (tango_b200/csrc/tng_ptx.cuh), the polynomial 2^x that takes part of the flash-attention softmax's
exponentials off MUFU: a torch fp32 statement that follows the device code operation by operation (the same roundings,
the same FMA order), held to float64 exp2 on a dense grid over [-126, 0] and at the edges the softmax reaches.
test_attention_exp2_gpu.py requires the device function to reproduce this statement bit for bit."""
import math

import torch

# the Horner coefficients of tng_ptx.cuh, degree 4 down to 1 (the constant term is 1)
C4, C3, C2, C1 = (float.fromhex(h) for h in ("0x1.b7ea5cp-7", "0x1.abfe7ep-5", "0x1.ee2374p-3", "0x1.62d6d0p-1"))
REL_BOUND = 2.0 ** -16   # 2^7 below the bf16 rounding of P


def fma_f32(a, b, c):
    """fp32 fused multiply-add, rounded once to nearest-even, for fp32 tensors (or Python floats)."""
    a, b, c = (torch.as_tensor(v, dtype=torch.float32) for v in (a, b, c))
    p = a.double() * b.double()          # exact: 24 + 24 significant bits
    cd = c.double()
    s = p + cd
    bp = s - p
    e = (p - (s - bp)) + (cd - bp)       # s + e == a * b + c exactly (TwoSum)
    rd = s.float().double()
    # Rounding s instead of s + e to fp32 can only go wrong when s is exactly halfway between two fp32 values: then
    # `other`, the second neighbour, is an fp32 value, and the sign of e decides.
    other = 2.0 * s - rd
    tie = (other != rd) & (other.float().double() == other) & (e != 0)
    fixed = torch.where(e > 0, torch.maximum(rd, other), torch.minimum(rd, other))
    return torch.where(tie, fixed, rd).float()


def ex2_poly_ref(x):
    """tng::ex2_poly on an fp32 tensor."""
    x = torch.clamp_min(x.float(), -127.0)                    # fmaxf(x, -127)
    n = torch.floor(x)                                         # __fadd_rd(x, 1.5 * 2^23) - 1.5 * 2^23
    f = x - n
    p = fma_f32(C4, f, C3)
    p = fma_f32(p, f, C2)
    p = fma_f32(p, f, C1)
    p = fma_f32(p, f, 1.0)
    scale = ((n.to(torch.int32) + 127) << 23).view(torch.float32)   # 2^n, +0 for n = -127
    return p * scale


def dense_grid():
    """[-126, 0] in 2^22 + 1 even steps, the fp32 neighbours of every integer in it, and seeded random fp32 values."""
    g = torch.linspace(-126.0, 0.0, 2 ** 22 + 1, dtype=torch.float64).float()
    ints = torch.arange(-126, 1, dtype=torch.float32)
    near = torch.cat([torch.nextafter(ints, torch.full_like(ints, -math.inf)),
                      torch.nextafter(ints, torch.full_like(ints, math.inf)), ints])
    near = near[(near >= -126.0) & (near <= 0.0)]
    rnd = -126.0 * torch.rand(1 << 20, generator=torch.Generator().manual_seed(0), dtype=torch.float64).float()
    small = -torch.logspace(-40, 0, 4097, dtype=torch.float64).float()   # tiny scores next to the row maximum
    return torch.cat([g, near, rnd, small[small.abs() > 0]])


EDGES = [   # (fp32 input, the exact result of ex2.approx.ftz): masked keys, flush to zero below -126, the row maximum
    (-math.inf, 0.0),
    (-2.0 ** 100, 0.0),
    (-200.0, 0.0),
    (-127.5, 0.0),
    (-127.0, 0.0),
    (-126.75, 0.0),
    (float(torch.nextafter(torch.tensor(-126.0), torch.tensor(-math.inf))), 0.0),
    (-126.0, 2.0 ** -126),
    (-64.0, 2.0 ** -64),
    (-1.0, 0.5),
    (-0.0, 1.0),
    (0.0, 1.0),
]


def edge_inputs():
    return torch.tensor([x for x, _ in EDGES], dtype=torch.float32)


def test_fma_f32_rounds_once():
    # (1 + 2^-23) * (1 - 2^-23) 2^-24 + (1 + 2^-23) = 1 + 3 * 2^-24 - 2^-70: float64 rounds the sum to the fp32 tie
    # 1 + 3 * 2^-24, which goes to the even 1 + 2^-22, while the exact value lies below the tie: 1 + 2^-23
    a, b, c = 1.0 + 2.0 ** -23, (1.0 - 2.0 ** -23) * 2.0 ** -24, 1.0 + 2.0 ** -23
    assert float(torch.tensor(a * b + c).float()) == 1.0 + 2.0 ** -22
    assert float(fma_f32(a, b, c)) == 1.0 + 2.0 ** -23
    assert float(fma_f32(1.0, 2.0 ** -24, 1.0)) == 1.0                          # exactly the tie: to even
    assert float(fma_f32(1.0 + 2.0 ** -23, 2.0 ** -24, 1.0)) == 1.0 + 2.0 ** -23   # above the tie


def test_ex2_poly_relative_error_on_dense_grid():
    x = dense_grid()
    got = ex2_poly_ref(x).double()
    want = torch.exp2(x.double())
    rel = ((got - want).abs() / want).max().item()
    assert rel <= REL_BOUND, f"max relative error {rel:.3e} = 2^{math.log2(rel):.2f}"
    assert rel <= 2.0 ** -18, f"max relative error {rel:.3e} = 2^{math.log2(rel):.2f} (the stated bound is 2^-18)"


def test_ex2_poly_edges():
    x = edge_inputs()
    got = ex2_poly_ref(x)
    for (xi, want), gi in zip(EDGES, got.tolist()):
        assert gi == want, (xi, gi, want)
        if want == 0.0:
            assert math.copysign(1.0, gi) == 1.0, f"{xi} must give +0"


def test_ex2_poly_is_monotone():
    # the softmax only needs P >= 0 and no reordering of scores; check it is non-decreasing on a sorted grid
    x = torch.linspace(-126.0, 0.0, 1 << 20, dtype=torch.float64).float()
    y = ex2_poly_ref(x)
    assert bool((y[1:] >= y[:-1]).all())
