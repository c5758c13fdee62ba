"""tng::ex2_poly on the H100 against its torch statement (test_attention_exp2_cpu.py), bit for bit, on the same inputs:
the dense grid over [-126, 0] and the edges. The device function is compiled from tng_ptx.cuh with the library's own
nvcc flags into a small test library in a temporary directory."""
import ctypes
import os
import subprocess

import pytest
import torch

from test_attention_exp2_cpu import EDGES, dense_grid, edge_inputs, ex2_poly_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNELS = r"""
#include "tng_ptx.cuh"
__global__ void ex2_poly_kernel(const float* x, float* y, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = tng::ex2_poly(x[i]);
}
__global__ void ex2_approx_kernel(const float* x, float* y, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = tng::ex2_approx(x[i]);
}
extern "C" int run_ex2(int poly, const float* x, float* y, int n) {
  if (poly) ex2_poly_kernel<<<(n + 255) / 256, 256>>>(x, y, n);
  else ex2_approx_kernel<<<(n + 255) / 256, 256>>>(x, y, n);
  return static_cast<int>(cudaDeviceSynchronize());
}
"""


@pytest.fixture(scope="module")
def ex2_lib(tmp_path_factory):
    from tango_b200 import build as b
    d = tmp_path_factory.mktemp("ex2_poly")
    src, so = d / "ex2.cu", d / "libex2.so"
    src.write_text(KERNELS)
    cmd = [b._nvcc(), *b.NVCC_FLAGS, "-shared", "-I", b.CSRC, str(src), "-o", str(so)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    lib = ctypes.CDLL(str(so))
    lib.run_ex2.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    lib.run_ex2.restype = ctypes.c_int
    return lib


def run(lib, poly, x):
    xd = x.contiguous().cuda()
    yd = torch.empty_like(xd)
    assert lib.run_ex2(int(poly), xd.data_ptr(), yd.data_ptr(), xd.numel()) == 0
    return yd.cpu()


def test_ex2_poly_bit_identical_to_torch_statement(cuda, ex2_lib):
    x = torch.cat([dense_grid(), edge_inputs()])
    got, want = run(ex2_lib, True, x), ex2_poly_ref(x)
    same = got.view(torch.int32) == want.view(torch.int32)
    bad = (~same).nonzero().flatten()[:5]
    assert bool(same.all()), [(x[i].item(), got[i].item(), want[i].item()) for i in bad]


def test_ex2_poly_edges_match_ex2_approx(cuda, ex2_lib):
    x = edge_inputs()
    poly, approx = run(ex2_lib, True, x), run(ex2_lib, False, x)
    for (xi, want), p, a in zip(EDGES, poly.tolist(), approx.tolist()):
        assert p == want, (xi, p, want)
        if want in (0.0, 1.0):   # -inf, below -126 and 0: where the softmax relies on the exact value
            assert a == want, (xi, a, want)
