"""CPU restatement of the diffusers fork's DPMSolverMultistepScheduler (TEST INFRASTRUCTURE ONLY).

Follows /root/reference/mustango/diffusers/src/diffusers/schedulers/scheduling_dpmsolver_multistep.py operation by
operation in torch fp32 on the CPU, like oracle/schedulers.py does for DDPM / DDIM, so the results are bit-identical to
the reference run on CPU. `reference_class()` loads the fork's own class through oracle/refshim.py.
"""
from __future__ import annotations

import numpy as np
import torch

from .schedulers import make_betas


def reference_class():
    """The fork's DPMSolverMultistepScheduler (scheduling_dpmsolver_multistep.py), unmodified."""
    from . import refshim
    refshim.install()
    from diffusers.schedulers.scheduling_dpmsolver_multistep import DPMSolverMultistepScheduler
    return DPMSolverMultistepScheduler


class OracleDPMSolverMultistep:
    """scheduling_dpmsolver_multistep.py:124-495 (no thresholding), op by op in torch fp32 on the CPU."""

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, solver_order=2, prediction_type="epsilon", algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True, **_ignored):
        self.T = num_train_timesteps
        if trained_betas is not None:
            self.betas = torch.tensor(trained_betas, dtype=torch.float32)
        else:
            self.betas = make_betas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)                       # :157-160
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.init_noise_sigma = 1.0
        self.order_k = solver_order
        self.prediction_type = prediction_type
        self.algorithm_type = "dpmsolver++" if algorithm_type == "deis" else algorithm_type
        self.solver_type = "midpoint" if solver_type in ("logrho", "bh1", "bh2") else solver_type
        self.lower_order_final = lower_order_final
        self.num_inference_steps = None
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0

    def set_timesteps(self, n):
        """:185-206."""
        self.num_inference_steps = n
        ts = np.linspace(0, self.T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts)
        self.model_outputs = [None] * self.order_k
        self.lower_order_nums = 0

    def convert(self, mo, t, sample):
        """:243-281."""
        a, s = self.alpha_t[t], self.sigma_t[t]
        if self.algorithm_type == "dpmsolver++":
            if self.prediction_type == "epsilon":
                return (sample - s * mo) / a
            if self.prediction_type == "sample":
                return mo
            return a * sample - s * mo
        if self.prediction_type == "epsilon":
            return mo
        if self.prediction_type == "sample":
            return (sample - a * mo) / s
        return a * mo + s * sample

    def first(self, m, s0, t, x):
        """:305-313."""
        h = self.lambda_t[t] - self.lambda_t[s0]
        a_t, a_s = self.alpha_t[t], self.alpha_t[s0]
        g_t, g_s = self.sigma_t[t], self.sigma_t[s0]
        if self.algorithm_type == "dpmsolver++":
            return (g_t / g_s) * x - (a_t * (torch.exp(-h) - 1.0)) * m
        return (a_t / a_s) * x - (g_t * (torch.exp(h) - 1.0)) * m

    def second(self, ms, ts, t, x):
        """:336-372."""
        s0, s1 = ts[-1], ts[-2]
        m0, m1 = ms[-1], ms[-2]
        lt, l0, l1 = self.lambda_t[t], self.lambda_t[s0], self.lambda_t[s1]
        a_t, a_0 = self.alpha_t[t], self.alpha_t[s0]
        g_t, g_0 = self.sigma_t[t], self.sigma_t[s0]
        h, h_0 = lt - l0, l0 - l1
        r0 = h_0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        if self.algorithm_type == "dpmsolver++":
            if self.solver_type == "midpoint":
                return (g_t / g_0) * x - (a_t * (torch.exp(-h) - 1.0)) * D0 - 0.5 * (a_t * (torch.exp(-h) - 1.0)) * D1
            return (g_t / g_0) * x - (a_t * (torch.exp(-h) - 1.0)) * D0 + (a_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1
        if self.solver_type == "midpoint":
            return (a_t / a_0) * x - (g_t * (torch.exp(h) - 1.0)) * D0 - 0.5 * (g_t * (torch.exp(h) - 1.0)) * D1
        return (a_t / a_0) * x - (g_t * (torch.exp(h) - 1.0)) * D0 - (g_t * ((torch.exp(h) - 1.0) / h - 1.0)) * D1

    def third(self, ms, ts, t, x):
        """:395-427."""
        s0, s1, s2 = ts[-1], ts[-2], ts[-3]
        m0, m1, m2 = ms[-1], ms[-2], ms[-3]
        lt, l0, l1, l2 = self.lambda_t[t], self.lambda_t[s0], self.lambda_t[s1], self.lambda_t[s2]
        a_t, a_0 = self.alpha_t[t], self.alpha_t[s0]
        g_t, g_0 = self.sigma_t[t], self.sigma_t[s0]
        h, h_0, h_1 = lt - l0, l0 - l1, l1 - l2
        r0, r1 = h_0 / h, h_1 / h
        D0 = m0
        D1_0, D1_1 = (1.0 / r0) * (m0 - m1), (1.0 / r1) * (m1 - m2)
        D1 = D1_0 + (r0 / (r0 + r1)) * (D1_0 - D1_1)
        D2 = (1.0 / (r0 + r1)) * (D1_0 - D1_1)
        if self.algorithm_type == "dpmsolver++":
            return ((g_t / g_0) * x - (a_t * (torch.exp(-h) - 1.0)) * D0 + (a_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1
                    - (a_t * ((torch.exp(-h) - 1.0 + h) / h ** 2 - 0.5)) * D2)
        return ((a_t / a_0) * x - (g_t * (torch.exp(h) - 1.0)) * D0 - (g_t * ((torch.exp(h) - 1.0) / h - 1.0)) * D1
                - (g_t * ((torch.exp(h) - 1.0 - h) / h ** 2 - 0.5)) * D2)

    def step(self, model_output, t, sample, noise=None):
        """:429-495 (`noise` is accepted for the oracle loop's call signature and ignored: nothing is drawn)."""
        ts = self.timesteps
        hits = (ts == t).nonzero()
        i = len(ts) - 1 if len(hits) == 0 else hits.item()
        n = len(ts)
        prev_t = 0 if i == n - 1 else ts[i + 1]
        low = self.lower_order_final and n < 15
        m = self.convert(model_output, t, sample)
        for k in range(self.order_k - 1):
            self.model_outputs[k] = self.model_outputs[k + 1]
        self.model_outputs[-1] = m
        if self.order_k == 1 or self.lower_order_nums < 1 or (low and i == n - 1):
            x = self.first(m, t, prev_t, sample)
        elif self.order_k == 2 or self.lower_order_nums < 2 or (low and i == n - 2):
            x = self.second(self.model_outputs, [ts[i - 1], t], prev_t, sample)
        else:
            x = self.third(self.model_outputs, [ts[i - 2], ts[i - 1], t], prev_t, sample)
        if self.lower_order_nums < self.order_k:
            self.lower_order_nums += 1
        return x
