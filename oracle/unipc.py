"""CPU restatement of the diffusers fork's UniPCMultistepScheduler (TEST INFRASTRUCTURE ONLY).

Follows /root/reference/mustango/diffusers/src/diffusers/schedulers/scheduling_unipc_multistep.py in torch fp32 on the
CPU, like oracle/dpm_solver.py does for the DPM-Solver, so the results are bit-identical to the reference run on CPU.
`reference_class()` loads the fork's own class through oracle/refshim.py.
"""
from __future__ import annotations

import numpy as np
import torch

from .schedulers import make_betas


def reference_class():
    """The fork's UniPCMultistepScheduler (scheduling_unipc_multistep.py), unmodified."""
    from . import refshim
    refshim.install()
    from diffusers.schedulers.scheduling_unipc_multistep import UniPCMultistepScheduler
    return UniPCMultistepScheduler


class OracleUniPCMultistep:
    """scheduling_unipc_multistep.py:126-572 (no thresholding, no solver_p), in torch fp32 on the CPU."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, solver_order=2, prediction_type="epsilon", predict_x0=True, solver_type="bh2",
                 lower_order_final=True, disable_corrector=(), **_ignored):
        self.T = num_train_timesteps
        if trained_betas is not None:
            self.betas = torch.tensor(trained_betas, dtype=torch.float32)
        else:
            self.betas = make_betas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.alphas_cumprod = torch.cumprod(1.0 - self.betas, dim=0)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.init_noise_sigma = 1.0
        self.k = solver_order
        self.prediction_type = prediction_type
        self.predict_x0 = predict_x0
        self.bh2 = solver_type == "bh2"          # midpoint / heun / logrho are bh1 in the fork
        self.lower_order_final = lower_order_final
        self.disable_corrector = list(disable_corrector)
        self.model_outputs = [None] * solver_order
        self.ts_hist = [None] * solver_order
        self.lower_order_nums = 0
        self.last_sample = None
        self.this_order = None

    def set_timesteps(self, n):
        self.num_inference_steps = n
        self.timesteps = torch.from_numpy(np.linspace(0, self.T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64))
        self.model_outputs = [None] * self.k
        self.lower_order_nums = 0
        self.last_sample = None

    def convert(self, mo, t, x):
        a, s = self.alpha_t[t], self.sigma_t[t]
        if self.predict_x0:
            return {"epsilon": lambda: (x - s * mo) / a, "sample": lambda: mo,
                    "v_prediction": lambda: a * x - s * mo}[self.prediction_type]()
        return {"epsilon": lambda: mo, "sample": lambda: (x - a * mo) / s,
                "v_prediction": lambda: a * mo + s * x}[self.prediction_type]()

    def _terms(self, s0, t, order):
        """h-dependent scalars, the ratios r_k and the differences D_k of the history against its newest entry."""
        lt, l0 = self.lambda_t[t], self.lambda_t[s0]
        h = lt - l0
        m0 = self.model_outputs[-1]
        rks, D = [], []
        for j in range(1, order):
            rk = (self.lambda_t[self.ts_hist[-(j + 1)]] - l0) / h
            rks.append(rk)
            D.append((self.model_outputs[-(j + 1)] - m0) / rk)
        rks = torch.tensor(rks + [1.0])
        hh = -h if self.predict_x0 else h
        hphi1 = torch.expm1(hh)
        bh = torch.expm1(hh) if self.bh2 else hh
        hphik = hphi1 / hh - 1
        R, b, fac = [], [], 1
        for j in range(1, order + 1):
            R.append(torch.pow(rks, j - 1))
            b.append(hphik * fac / bh)
            fac *= j + 1
            hphik = hphik / hh - 1 / fac
        if self.predict_x0:
            cx, cm, cb = self.sigma_t[t] / self.sigma_t[s0], self.alpha_t[t] * hphi1, self.alpha_t[t] * bh
        else:
            cx, cm, cb = self.alpha_t[t] / self.alpha_t[s0], self.sigma_t[t] * hphi1, self.sigma_t[t] * bh
        return cx, cm, cb, torch.stack(R), torch.tensor(b), D, m0

    def corrector(self, m_t, t, x_last):
        cx, cm, cb, R, b, D, m0 = self._terms(self.ts_hist[-1], t, self.this_order)
        rho = torch.tensor([0.5]) if self.this_order == 1 else torch.linalg.solve(R, b)
        res = torch.einsum("k,bkchw->bchw", rho[:-1], torch.stack(D, dim=1)) if D else 0
        return cx * x_last - cm * m0 - cb * (res + rho[-1] * (m_t - m0))

    def predictor(self, t, x, order):
        cx, cm, cb, R, b, D, m0 = self._terms(self.ts_hist[-1], t, order)
        res = 0
        if D:
            rho = torch.tensor([0.5]) if order == 2 else torch.linalg.solve(R[:-1, :-1], b[:-1])
            res = torch.einsum("k,bkchw->bchw", rho, torch.stack(D, dim=1))
        return cx * x - cm * m0 - cb * res

    def step(self, model_output, t, sample, noise=None):
        """(`noise` is accepted for the oracle loops' call signature and ignored: nothing is drawn.)"""
        hits = (self.timesteps == t).nonzero()
        i = len(self.timesteps) - 1 if len(hits) == 0 else hits.item()
        n = len(self.timesteps)
        m = self.convert(model_output, t, sample)
        if i > 0 and (i - 1) not in self.disable_corrector and self.last_sample is not None:
            sample = self.corrector(m, t, self.last_sample)
        t_next = 0 if i == n - 1 else self.timesteps[i + 1]
        self.model_outputs = self.model_outputs[1:] + [m]
        self.ts_hist = self.ts_hist[1:] + [t]
        order = min(self.k, n - i) if self.lower_order_final else self.k
        self.this_order = min(order, self.lower_order_nums + 1)
        self.last_sample = sample
        x = self.predictor(t_next, sample, self.this_order)
        if self.lower_order_nums < self.k:
            self.lower_order_nums += 1
        return x


def fma32(a, b, c):
    """fp32 fma(a, b, c) with one rounding, elementwise: a * b is exact in fp64 and the fp64 sum is rounded to odd
    (its TwoSum error term decides), which makes the final rounding to fp32 correct."""
    p, cd = a.double() * b.double(), c.double()
    s = p + cd
    bv = s - p
    err = (p - (s - bv)) + (cd - bv)
    even = (s.view(torch.int64) & 1) == 0
    toward = torch.where(err > 0, torch.full_like(s, float("inf")), torch.full_like(s, float("-inf")))
    return torch.where((err != 0) & even, torch.nextafter(s, toward), s).float()
