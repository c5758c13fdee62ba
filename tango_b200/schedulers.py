"""DDPM / DDIM / multistep DPM-Solver / UniPC schedulers with the reference's interface; the update itself runs in one
fused CUDA kernel.

Mirrors diffusers' DDPMScheduler / DDIMScheduler as Tango uses them
(/root/reference/mustango/diffusers/src/diffusers/schedulers/scheduling_ddpm.py:122-349,
scheduling_ddim.py:132-359; call sites models.py:224-249, tango.py:36): `set_timesteps`, `timesteps`,
`init_noise_sigma`, `order`, `scale_model_input`, `step(...).prev_sample`, `config`. DPMSolverMultistepScheduler
(scheduling_dpmsolver_multistep.py:57-535) and UniPCMultistepScheduler (scheduling_unipc_multistep.py:80-572) are the
opt-in few-step samplers; their updates run in tng_dpm_step and tng_unipc_step (below).

All per-step scalars are computed on the host with the reference's own fp32 torch ops (same association order),
packed into a [num_steps, 10] coefficient table and shipped to the device once per timestep grid; the kernel
(tng_sched_step) then evaluates  x0 = (c0*s + c1*v)/c9, prev = c2*x0 + c3*s + c7*(c5*s + c6*v) + c4*noise  with
un-fused multiplies/adds, which reproduces the reference CPU arithmetic bit for bit and removes the two host syncs
per step of the reference (SURVEY.md §1).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional

import numpy as np
import torch

from . import lib as L

# stabilityai/stable-diffusion-2-1 `scheduler/scheduler_config.json` — what Tango loads (tango.py:36, models.py:80-81).
# The JSON is not in the reference tree (SURVEY.md F6); these are its published values and every field can be overridden.
SD21_SCHEDULER_CONFIG = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012,
                             beta_schedule="scaled_linear", prediction_type="v_prediction", clip_sample=False,
                             set_alpha_to_one=False, steps_offset=1, skip_prk_steps=True, trained_betas=None)

NCOEF = 10


class SchedulerOutput(SimpleNamespace):
    pass


class _Config(dict):
    __getattr__ = dict.__getitem__


def _betas(num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas=None):
    if trained_betas is not None:
        return torch.tensor(trained_betas, dtype=torch.float32)
    if beta_schedule == "linear":
        return torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    if beta_schedule == "scaled_linear":
        return torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    raise NotImplementedError(f"{beta_schedule} is not implemented")


class _SchedulerBase:
    order = 1

    def __init__(self, **cfg):
        self.config = _Config(cfg)
        self.betas = _betas(cfg["num_train_timesteps"], cfg["beta_start"], cfg["beta_end"], cfg["beta_schedule"],
                            cfg.get("trained_betas"))
        self.alphas = 1.0 - self.betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.init_noise_sigma = 1.0
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.from_numpy(np.arange(0, cfg["num_train_timesteps"])[::-1].copy().astype(np.int64))
        self._t_list: Optional[list] = None
        self._t_index: dict = {}
        self._tables: dict = {}   # (kind, grid, t_start) -> (host table, DPM loop orders or None, {device: copy})

    @classmethod
    def from_pretrained(cls, name: str = "stabilityai/stable-diffusion-2-1", subfolder: str = "scheduler", **overrides):
        """The reference downloads the SD-2.1 scheduler JSON from the hub (tango.py:36, models.py:80-81). Offline:
        a local directory is read (`<name>/<subfolder>/scheduler_config.json` or `<name>/scheduler_config.json`);
        `stabilityai/stable-diffusion-2-1` (or None) maps to its published values; any other name is refused rather
        than silently sampled with the wrong betas / prediction type."""
        import json
        import os
        base = dict(SD21_SCHEDULER_CONFIG)
        if name is not None and os.path.isdir(str(name)):
            for cand in (os.path.join(name, subfolder or "", "scheduler_config.json"), os.path.join(name, "scheduler_config.json")):
                if os.path.exists(cand):
                    with open(cand) as f:
                        base.update({k: v for k, v in json.load(f).items() if not k.startswith("_")})
                    break
            else:
                raise FileNotFoundError(f"no scheduler_config.json under '{name}'")
        elif name not in (None, "stabilityai/stable-diffusion-2-1"):
            raise ValueError(f"scheduler '{name}' is not reachable offline: pass a local directory holding its "
                             "scheduler_config.json (only stabilityai/stable-diffusion-2-1 is built in)")
        base.update(overrides)
        return cls.from_config(base)

    @classmethod
    def from_config(cls, config: dict, **overrides):
        """diffusers' `from_config`: the keys this scheduler's constructor accepts are kept, the rest dropped, so
        `DPMSolverMultistepScheduler.from_config(ddpm.config)` builds a DPM-Solver on the DDPM's betas."""
        cfg = dict(config, **overrides)
        return cls(**{k: v for k, v in cfg.items() if k in cls._ACCEPTED})

    def __len__(self):
        return self.config["num_train_timesteps"]

    def scale_model_input(self, sample, timestep=None):
        return sample

    # ---------------------------------------------------------------------------------------------------------
    def _grid(self, n: int) -> np.ndarray:
        T = self.config["num_train_timesteps"]
        if n > T:
            raise ValueError(
                f"`num_inference_steps`: {n} cannot be larger than `self.config.train_timesteps`: {T} as the unet"
                f" model trained with this scheduler can only handle maximal {T} timesteps.")
        ratio = T // n
        return (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64)

    def _finish_set_timesteps(self, device):
        self._t_list = [int(t) for t in self.timesteps.tolist()]
        self._t_index = {t: i for i, t in enumerate(self._t_list)}
        if device is not None:
            self.timesteps = self.timesteps.to(device)
        self.coefficient_table(device)

    def _table(self, kind: str, device=None, t_start: int = 0):
        """(table, loop orders) of the current grid for a loop entered at timesteps[t_start]; row i belongs to
        timesteps[i]. kind "coef" is the update's coefficient table, "blend" the add_noise rows. Each (kind, grid,
        t_start) is computed once (~40 tiny fp32 torch ops per row) and copied to each device once; `device` None
        gives the host table."""
        if self._t_list is None:
            self._finish_set_timesteps(None)
        key = (kind, tuple(self._t_list), t_start)
        if key not in self._tables:
            rows, orders = self._table_rows(kind, t_start)
            self._tables[key] = (torch.stack(rows).contiguous(), orders, {})
        host, orders, dev = self._tables[key]
        if device is None:
            return host, orders
        d = str(torch.device(device))
        if d not in dev:
            dev[d] = host.to(device)
        return dev[d], orders

    def _table_rows(self, kind: str, t_start: int):
        """The rows of table `kind` and the loop orders they belong to (None: they do not depend on the order)."""
        row = self._blend_row if kind == "blend" else self._coefficients
        return [row(t) for t in self._t_list], None

    def loop_table(self, device, t_start: int = 0) -> torch.Tensor:
        """Coefficient table of a loop that runs timesteps[t_start:] (row i belongs to timesteps[i]); only the
        multistep DPM-Solver's rows depend on where the loop starts."""
        return self.coefficient_table(device)

    def get_timesteps(self, num_inference_steps: int, strength: float):
        """Img2img's `get_timesteps` (pipeline_stable_diffusion_img2img.py:509-516) on the grid of `set_timesteps`:
        returns (t_start, timesteps[t_start:]). `strength` outside [0, 1], or so small that no step runs, raises."""
        if strength < 0 or strength > 1:
            raise ValueError(f"The value of strength should in [0.0, 1.0] but is {strength}")
        init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
        if init_timestep == 0:
            raise ValueError(f"strength {strength} with {num_inference_steps} steps runs no denoising step "
                             f"(int({num_inference_steps} * {strength}) == 0): raise the strength or the step count")
        t_start = max(num_inference_steps - init_timestep, 0)
        return t_start, self.timesteps[t_start:]

    def _blend_row(self, t: int) -> torch.Tensor:
        """add_noise's fp32 scalars at timestep t (scheduling_ddpm.py:361-366): alphas_cumprod[t] ** 0.5 and
        (1 - alphas_cumprod[t]) ** 0.5."""
        a = self.alphas_cumprod[torch.tensor([int(t)])]
        return torch.cat([a ** 0.5, (1 - a) ** 0.5]).float()

    def blend_table(self, device=None) -> torch.Tensor:
        """[num_steps, 2] fp32 add_noise coefficients of the current grid (row i belongs to timesteps[i]): the
        coefficient rows of tng_latent_blend."""
        return self._table("blend", device)[0]

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps) -> torch.Tensor:
        """scheduling_ddpm.py:351-372 (DDIM and DPM-Solver share it) for fp32 CUDA tensors of shape (B, C, ...):
        sqrt(alphas_cumprod[t]) * original_samples + sqrt(1 - alphas_cumprod[t]) * noise, on tng_latent_blend.
        `timesteps` holds one timestep or one per sample."""
        L.require_cuda(original_samples, noise)   # no CPU fallback
        if original_samples.shape != noise.shape or original_samples.dim() < 2:
            raise ValueError(f"add_noise: original_samples {tuple(original_samples.shape)} and noise "
                             f"{tuple(noise.shape)} must share one (B, C, ...) shape")
        ts = [int(t) for t in torch.as_tensor(timesteps).reshape(-1).tolist()]
        B, Cc = original_samples.shape[:2]
        if len(ts) not in (1, B):
            raise ValueError(f"add_noise: {len(ts)} timesteps for a batch of {B}")
        HW = original_samples[0, 0].numel()
        x0, nz = original_samples.float().contiguous(), noise.float().contiguous()
        out = torch.empty_like(x0)
        rows = torch.stack([self._blend_row(t) for t in ts]).to(x0.device)
        if len(ts) == 1:
            L.latent_blend(x0, nz, None, rows[0], out, B=B, Cc=Cc, HW=HW)
        else:
            for b in range(B):
                L.latent_blend(x0[b], nz[b], None, rows[b], out[b], B=1, Cc=Cc, HW=HW)
        return out

    def _loop_step(self, i: int, model_out, cfg: bool, guidance: float, sample, noise, coef, next_in, bufs, *, B, Cc,
                   HW, split_off):
        """Step i of AudioDiffusion.inference: one fused CFG + update + next-UNet-input launch, `sample` updated in
        place. `bufs` holds the loop's persistent buffers of this shape."""
        L.sched_step(model_out, cfg, guidance, sample, noise, coef[i], sample, next_in, B=B, Cc=Cc, HW=HW,
                     split_off=split_off)

    def timestep_at(self, i: int) -> int:
        """Host copy of timesteps[i] (no device sync)."""
        return self._t_list[i]

    def coefficient_table(self, device=None) -> torch.Tensor:
        """[num_steps, 10] fp32 table (row i belongs to timesteps[i])."""
        return self._table("coef", device)[0]

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None,
             variance_noise: Optional[torch.Tensor] = None, return_dict: bool = True, **_unused):
        """x_t -> x_{t-1} for NCHW fp32 CUDA tensors (reference layout). Noise comes from the torch RNG exactly as
        in the reference (randn of model_output's shape when t > 0) unless `variance_noise` is given."""
        L.require_cuda(model_output)   # no CPU fallback
        i = self._t_index.get(int(timestep))
        if i is None:   # a timestep outside the grid (the reference allows it) gets a row of its own
            coef = self._coefficients(int(timestep)).to(sample.device)
        else:
            coef = self.coefficient_table(sample.device)[i]
        B, Cc, H, W = sample.shape
        noise = None
        if self._needs_noise(int(timestep)):
            noise = variance_noise
            if noise is None:
                noise = torch.randn(model_output.shape, generator=generator, device=model_output.device,
                                    dtype=model_output.dtype)
            noise = noise.contiguous().float()
        mo = model_output.float().permute(0, 2, 3, 1).contiguous().view(B * H * W, Cc)  # channels-last rows
        prev = torch.empty_like(sample, dtype=torch.float32)
        L.sched_step(mo, False, 1.0, sample.contiguous().float(), noise, coef.contiguous(), prev, None, B=B, Cc=Cc,
                     HW=H * W)
        if not return_dict:
            return (prev,)
        return SchedulerOutput(prev_sample=prev)


class DDPMScheduler(_SchedulerBase):
    _ACCEPTED = ("num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "trained_betas", "variance_type",
                 "clip_sample", "prediction_type", "clip_sample_range")

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, variance_type="fixed_small", clip_sample=True, prediction_type="epsilon",
                 clip_sample_range=1.0):
        if variance_type != "fixed_small":
            raise NotImplementedError("only variance_type='fixed_small' (Tango's) is implemented")
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, trained_betas=trained_betas, variance_type=variance_type,
                         clip_sample=clip_sample, prediction_type=prediction_type,
                         clip_sample_range=clip_sample_range)
        self.one = torch.tensor(1.0)
        self.variance_type = variance_type

    def set_timesteps(self, num_inference_steps: int, device=None):
        """scheduling_ddpm.py:184-204: t_i = (i * (T // N)) reversed, int64 (no steps_offset in this version)."""
        self.timesteps = torch.from_numpy(self._grid(num_inference_steps))
        self.num_inference_steps = num_inference_steps
        self._finish_set_timesteps(device)

    def _needs_noise(self, t: int) -> bool:
        return t > 0

    def _coefficients(self, t: int) -> torch.Tensor:
        """scheduling_ddpm.py:283-344 scalar arithmetic, same fp32 torch ops in the same order."""
        cfg = self.config
        n = self.num_inference_steps if self.num_inference_steps else cfg["num_train_timesteps"]
        prev_t = t - cfg["num_train_timesteps"] // n
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.one
        b_t = 1 - a_t
        b_prev = 1 - a_prev
        cur_alpha = a_t / a_prev
        cur_beta = 1 - cur_alpha
        one, zero = torch.tensor(1.0), torch.tensor(0.0)
        if cfg["prediction_type"] == "epsilon":
            c_x0_s, c_x0_m, c_div = one, -(b_t ** 0.5), a_t ** 0.5
        elif cfg["prediction_type"] == "sample":
            c_x0_s, c_x0_m, c_div = zero, one, one
        elif cfg["prediction_type"] == "v_prediction":
            c_x0_s, c_x0_m, c_div = a_t ** 0.5, -(b_t ** 0.5), one
        else:
            raise ValueError(f"prediction_type given as {cfg['prediction_type']} must be one of `epsilon`, `sample` or"
                             " `v_prediction`  for the DDPMScheduler.")
        c_prev_x0 = (a_prev ** 0.5 * cur_beta) / b_t
        c_prev_s = cur_alpha ** 0.5 * b_prev / b_t
        c_noise = zero
        if t > 0:
            var = (1 - a_prev) / (1 - a_t) * cur_beta   # _get_variance :206-224
            var = torch.clamp(var, min=1e-20)
            c_noise = var ** 0.5
        clip = torch.tensor(float(cfg["clip_sample_range"]) if cfg["clip_sample"] else 0.0)
        return torch.stack([c_x0_s, c_x0_m, c_prev_x0, c_prev_s, c_noise, zero, zero, zero, clip, c_div]).float()


class DDIMScheduler(_SchedulerBase):
    _ACCEPTED = ("num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "trained_betas", "clip_sample",
                 "set_alpha_to_one", "steps_offset", "prediction_type", "clip_sample_range")

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, clip_sample=True, set_alpha_to_one=True, steps_offset=0,
                 prediction_type="epsilon", clip_sample_range=1.0):
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, trained_betas=trained_betas, clip_sample=clip_sample,
                         set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset,
                         prediction_type=prediction_type, clip_sample_range=clip_sample_range)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]

    def set_timesteps(self, num_inference_steps: int, device=None):
        """scheduling_ddim.py:214-236: same grid as DDPM plus steps_offset."""
        self.timesteps = torch.from_numpy(self._grid(num_inference_steps)) + self.config["steps_offset"]
        self.num_inference_steps = num_inference_steps
        self._finish_set_timesteps(device)

    def _needs_noise(self, t: int) -> bool:
        return False  # eta = 0 (deterministic DDIM)

    def _coefficients(self, t: int) -> torch.Tensor:
        """scheduling_ddim.py:292-354 with eta = 0."""
        cfg = self.config
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the"
                             " scheduler")
        prev_t = t - cfg["num_train_timesteps"] // self.num_inference_steps
        a_t = self.alphas_cumprod[t]
        a_prev = self.alphas_cumprod[prev_t] if prev_t >= 0 else self.final_alpha_cumprod
        b_t = 1 - a_t
        one, zero = torch.tensor(1.0), torch.tensor(0.0)
        if cfg["prediction_type"] == "epsilon":
            c_x0_s, c_x0_m, c_div = one, -(b_t ** 0.5), a_t ** 0.5
            c_eps_s, c_eps_m = zero, one
        elif cfg["prediction_type"] == "v_prediction":
            c_x0_s, c_x0_m, c_div = a_t ** 0.5, -(b_t ** 0.5), one
            c_eps_s, c_eps_m = b_t ** 0.5, a_t ** 0.5
        else:
            raise ValueError(f"prediction_type given as {cfg['prediction_type']} must be one of `epsilon` or"
                             " `v_prediction` for the fused DDIM step")
        b_prev = 1 - a_prev
        variance = (b_prev / b_t) * (1 - a_t / a_prev)
        std = 0.0 * variance ** 0.5
        c_prev_eps = (1 - a_prev - std ** 2) ** 0.5
        c_prev_x0 = a_prev ** 0.5
        clip = torch.tensor(float(cfg["clip_sample_range"]) if cfg["clip_sample"] else 0.0)
        return torch.stack([c_x0_s, c_x0_m, c_prev_x0, zero, zero, c_eps_s, c_eps_m, c_prev_eps, clip,
                            c_div]).float()


NCOEF_DPM = 11
NCOEF_UNIPC = 18


class _MultistepBase(_SchedulerBase):
    """What the multistep ODE solvers (DPM-Solver, UniPC) share: the VP-type alpha / sigma / lambda schedule, the
    linspace timestep grid, the conversion of the model output to the solver's prediction, the persistent history
    slots of the sampling loop and the loop tables whose rows depend on the orders a loop takes."""

    def __init__(self, **cfg):
        super().__init__(**cfg)
        # VP-type noise schedule (scheduling_dpmsolver_multistep.py:157-160, scheduling_unipc_multistep.py:162-164)
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self._orders: list = []
        self._loop_orders: list = []

    def _set_grid(self, num_inference_steps: int):
        """linspace(0, T-1, n+1) rounded, reversed, last dropped (no steps_offset)."""
        self.num_inference_steps = num_inference_steps
        T = self.config["num_train_timesteps"]
        ts = np.linspace(0, T - 1, num_inference_steps + 1).round()[::-1][:-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts)

    def _needs_noise(self, t: int) -> bool:
        return False   # an ODE solver: nothing is drawn after the initial latents

    def _conversion(self, s0: int, data_prediction: bool):
        """{c_a, c_b, c_d} with converted = (c_a * sample + c_b * model_output) / c_d at timestep s0: the data
        prediction x0 (`data_prediction`) or the noise prediction, from the model's `prediction_type`."""
        one, zero = torch.tensor(1.0), torch.tensor(0.0)
        a_s0, sg_s0 = self.alpha_t[s0], self.sigma_t[s0]
        if data_prediction:
            return {"epsilon": (one, -sg_s0, a_s0), "sample": (zero, one, one),
                    "v_prediction": (a_s0, -sg_s0, one)}[self.config["prediction_type"]]
        return {"epsilon": (zero, one, one), "sample": (one, -a_s0, sg_s0),
                "v_prediction": (sg_s0, a_s0, one)}[self.config["prediction_type"]]

    def loop_table(self, device, t_start: int = 0) -> torch.Tensor:
        """The coefficient table of a loop entered at timesteps[t_start] (an edit): its rows follow the orders of a
        loop that starts there, which `_loop_step` then follows. t_start = 0 is the `set_timesteps` table itself."""
        tab, self._loop_orders = self._table("coef", device, t_start)
        return tab

    def _table_rows(self, kind: str, t_start: int):
        if kind != "coef":
            return super()._table_rows(kind, t_start)
        orders = self._loop_orders_from(len(self._t_list), t_start)
        return [self._coefficients_at(i, o) for i, o in enumerate(orders)], orders

    @staticmethod
    def _history(bufs, sample, count: int) -> list:
        """`count` persistent NCHW fp32 history slots of the loop, kept with the other buffers of this shape."""
        hist = bufs.__dict__.setdefault("solver_history", [])
        while len(hist) < count:
            hist.append(torch.zeros(sample.shape, device=sample.device, dtype=torch.float32))
        return hist


class DPMSolverMultistepScheduler(_MultistepBase):
    """Multistep DPM-Solver / DPM-Solver++ (scheduling_dpmsolver_multistep.py:57-535), for sampling in 20-25 steps.

    The CFG combine, `convert_model_output` and the order-1/2/3 update run as one tng_dpm_step launch. Its per-step
    scalars are computed here with the reference's own fp32 torch ops in the reference's order and packed into a
    [num_steps, 11] table (see include/tango_b200.h for the row): {c_a, c_b, c_d} convert the model output,
    m0 = (c_a * sample + c_b * v) / c_d; {c_s, c_0, c_1, c_2} weigh sample, D0, D1 and D2; then 1/r0, 1/r1,
    r0/(r0+r1) and 1/(r0+r1). Signs are folded into the coefficients, which IEEE arithmetic allows without changing a
    bit (x - y*z == x + (-y)*z). Row i uses the order that step i takes in a loop started by `set_timesteps`
    (`lower_order_nums` bookkeeping and the final-step rules, :464-490); `step` called out of that sequence gets a
    row of its own. Dynamic thresholding (per-sample quantile; unsuitable for latent diffusion per the fork's own
    docstring) is not implemented."""

    _ACCEPTED = ("num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "trained_betas", "solver_order",
                 "prediction_type", "thresholding", "dynamic_thresholding_ratio", "sample_max_value", "algorithm_type",
                 "solver_type", "lower_order_final")

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                 dynamic_thresholding_ratio=0.995, sample_max_value=1.0, algorithm_type="dpmsolver++",
                 solver_type="midpoint", lower_order_final=True):
        if thresholding:
            raise NotImplementedError("thresholding=True (dynamic thresholding) is not implemented for "
                                      "DPMSolverMultistepScheduler: it is unsuitable for latent diffusion")
        if algorithm_type == "deis":          # :166-170
            algorithm_type = "dpmsolver++"
        elif algorithm_type not in ("dpmsolver", "dpmsolver++"):
            raise NotImplementedError(f"{algorithm_type} does is not implemented for {self.__class__}")
        if solver_type in ("logrho", "bh1", "bh2"):   # :172-176
            solver_type = "midpoint"
        elif solver_type not in ("midpoint", "heun"):
            raise NotImplementedError(f"{solver_type} does is not implemented for {self.__class__}")
        if solver_order not in (1, 2, 3):
            raise ValueError(f"solver_order must be 1, 2 or 3, got {solver_order}")
        if prediction_type not in ("epsilon", "sample", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample`, or"
                             " `v_prediction` for the DPMSolverMultistepScheduler.")
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                         prediction_type=prediction_type, thresholding=thresholding,
                         dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                         algorithm_type=algorithm_type, solver_type=solver_type, lower_order_final=lower_order_final)
        self.model_outputs = [None] * solver_order
        self.lower_order_nums = 0

    def set_timesteps(self, num_inference_steps: int, device=None):
        """:185-206: linspace(0, T-1, n+1) rounded, reversed, last dropped (no steps_offset); resets the history."""
        self._set_grid(num_inference_steps)
        ts = self.timesteps
        self.model_outputs = [None] * self.config["solver_order"]
        self.lower_order_nums = 0
        self._orders = self._loop_orders_from(len(ts), 0)
        self._loop_orders = self._orders
        self._finish_set_timesteps(device)

    def _order_at(self, i: int, n: int, lower_order_nums: int) -> int:
        """The update order :476-487 picks at step index i of n with `lower_order_nums` earlier steps counted."""
        cfg = self.config
        low = cfg["lower_order_final"] and n < 15
        if cfg["solver_order"] == 1 or lower_order_nums < 1 or (low and i == n - 1):
            return 1
        if cfg["solver_order"] == 2 or lower_order_nums < 2 or (low and i == n - 2):
            return 2
        return 3

    def _loop_orders_from(self, n: int, t_start: int) -> list:
        """Orders of a loop over steps t_start..n-1 of an n-step grid: the fork counts `lower_order_nums` from the
        first `step` call, so the first executed step is order 1 and the next at most order 2, while the final-step
        rules still look at the whole grid (:464-490). Entries before t_start are the full loop's."""
        k = self.config["solver_order"]
        full = [self._order_at(i, n, min(i, k)) for i in range(n)]
        return full[:t_start] + [self._order_at(i, n, min(i - t_start, k)) for i in range(t_start, n)]

    def order_at(self, i: int) -> int:
        """Order of step i in a loop started by `set_timesteps`."""
        return self._orders[i]

    def _coefficients_at(self, i: int, order: int, timestep: Optional[int] = None) -> torch.Tensor:
        """The fp32 scalars of step index i at `order` (:243-281, :305-427, same torch ops in the same order).
        `timestep` overrides timesteps[i] for a step at a timestep outside the grid (the reference then takes the
        last index)."""
        cfg = self.config
        tl = self._t_list
        s0 = tl[i] if timestep is None else int(timestep)
        t = 0 if i == len(tl) - 1 else tl[i + 1]   # :463
        zero = torch.tensor(0.0)
        pp = cfg["algorithm_type"] == "dpmsolver++"
        c_a, c_b, c_d = self._conversion(s0, pp)
        lambda_t, lambda_s0 = self.lambda_t[t], self.lambda_t[s0]
        alpha_t, alpha_s0 = self.alpha_t[t], self.alpha_t[s0]
        sigma_t, sigma_s0 = self.sigma_t[t], self.sigma_t[s0]
        h = lambda_t - lambda_s0
        if pp:
            c_s, c_0 = sigma_t / sigma_s0, alpha_t * (torch.exp(-h) - 1.0)
        else:
            c_s, c_0 = alpha_t / alpha_s0, sigma_t * (torch.exp(h) - 1.0)
        c_1 = c_2 = inv_r0 = inv_r1 = w_r = inv_r01 = zero
        if order == 2:
            lambda_s1 = self.lambda_t[tl[i - 1]]
            h_0 = lambda_s0 - lambda_s1
            r0 = h_0 / h
            inv_r0 = 1.0 / r0
            if pp and cfg["solver_type"] == "midpoint":
                c_1 = -(0.5 * (alpha_t * (torch.exp(-h) - 1.0)))
            elif pp:
                c_1 = alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)
            elif cfg["solver_type"] == "midpoint":
                c_1 = -(0.5 * (sigma_t * (torch.exp(h) - 1.0)))
            else:
                c_1 = -(sigma_t * ((torch.exp(h) - 1.0) / h - 1.0))
        elif order == 3:
            lambda_s1, lambda_s2 = self.lambda_t[tl[i - 1]], self.lambda_t[tl[i - 2]]
            h_0, h_1 = lambda_s0 - lambda_s1, lambda_s1 - lambda_s2
            r0, r1 = h_0 / h, h_1 / h
            inv_r0, inv_r1 = 1.0 / r0, 1.0 / r1
            w_r, inv_r01 = r0 / (r0 + r1), 1.0 / (r0 + r1)
            if pp:
                c_1 = alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)
                c_2 = alpha_t * ((torch.exp(-h) - 1.0 + h) / h ** 2 - 0.5)
            else:
                c_1 = -(sigma_t * ((torch.exp(h) - 1.0) / h - 1.0))
                c_2 = sigma_t * ((torch.exp(h) - 1.0 - h) / h ** 2 - 0.5)
        return torch.stack([c_a, c_b, c_d, c_s, c_0, c_1, c_2, inv_r0, inv_r1, w_r, inv_r01]).float()

    def _loop_step(self, i: int, model_out, cfg: bool, guidance: float, sample, noise, coef, next_in, bufs, *, B, Cc,
                   HW, split_off):
        """Step i of AudioDiffusion.inference: the converted output goes to slot i mod k of k = solver_order
        history slots, the previous ones are read from slots i-1 and i-2 mod k."""
        k, order = self.config["solver_order"], self._loop_orders[i]
        hist = self._history(bufs, sample, k)
        m1 = hist[(i - 1) % k] if order >= 2 else None
        m2 = hist[(i - 2) % k] if order >= 3 else None
        L.dpm_step(model_out, cfg, guidance, sample, coef[i], order, hist[i % k], m1, m2, sample, next_in, B=B, Cc=Cc,
                   HW=HW, split_off=split_off)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, return_dict: bool = True, **_unused):
        """:429-495 for NCHW fp32 CUDA tensors: converts the model output, shifts it into `model_outputs`, takes the
        update of the order `lower_order_nums` and the final-step rules select, and counts `lower_order_nums`."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the"
                             " scheduler")
        L.require_cuda(model_output)   # no CPU fallback
        t = int(timestep)
        n = len(self._t_list)
        i = self._t_index.get(t, n - 1)
        k = self.config["solver_order"]
        order = self._order_at(i, n, self.lower_order_nums)
        if t == self._t_list[i] and order == self._orders[i]:
            coef = self.coefficient_table(sample.device)[i]
        else:
            coef = self._coefficients_at(i, order, t).to(sample.device)
        B, Cc, H, W = sample.shape
        m0 = torch.empty(sample.shape, device=sample.device, dtype=torch.float32)
        self.model_outputs = self.model_outputs[1:] + [m0]
        m1 = self.model_outputs[-2] if order >= 2 else None
        m2 = self.model_outputs[-3] if order >= 3 else None
        mo = model_output.float().permute(0, 2, 3, 1).contiguous().view(B * H * W, Cc)   # channels-last rows
        prev = torch.empty_like(sample, dtype=torch.float32)
        L.dpm_step(mo, False, 1.0, sample.contiguous().float(), coef, order, m0, m1, m2, prev, None, B=B, Cc=Cc,
                   HW=H * W)
        if self.lower_order_nums < k:
            self.lower_order_nums += 1
        if not return_dict:
            return (prev,)
        return SchedulerOutput(prev_sample=prev)


class UniPCMultistepScheduler(_MultistepBase):
    """Multistep UniPC (scheduling_unipc_multistep.py:80-572): the UniC corrector, then the UniP predictor, per step;
    built for 5-10 steps.

    The CFG combine, `convert_model_output`, the corrector and the predictor run as one tng_unipc_step launch. Its
    per-step scalars are computed here with the reference's own fp32 torch ops in the reference's order (the weights
    rho with its `torch.linalg.solve`) and packed into a [num_steps, 18] table (see include/tango_b200.h for the row):
    the conversion triple, then {c_x, c_m, c_b, r_0, r_1, rho_0, rho_1, rho_last} of the corrector and
    {c_x, c_m, c_b, r_0, r_1, rho_0, rho_1} of the predictor. Row i belongs to the (corrector, predictor) orders step i
    takes in a loop started by `set_timesteps` (or entered at an edit's t_start); `step` keeps the reference's state
    (`model_outputs`, `timestep_list`, `this_order`, `lower_order_nums`, `last_sample`) and computes the row that state
    calls for. As in the fork, `solver_type` midpoint / heun / logrho mean bh1. Dynamic thresholding and `solver_p`
    (another scheduler as the predictor) are not implemented."""

    _ACCEPTED = ("num_train_timesteps", "beta_start", "beta_end", "beta_schedule", "trained_betas", "solver_order",
                 "prediction_type", "thresholding", "dynamic_thresholding_ratio", "sample_max_value", "predict_x0",
                 "solver_type", "lower_order_final", "disable_corrector", "solver_p")

    def __init__(self, num_train_timesteps=1000, beta_start=0.0001, beta_end=0.02, beta_schedule="linear",
                 trained_betas=None, solver_order=2, prediction_type="epsilon", thresholding=False,
                 dynamic_thresholding_ratio=0.995, sample_max_value=1.0, predict_x0=True, solver_type="bh2",
                 lower_order_final=True, disable_corrector=(), solver_p=None):
        if thresholding:
            raise NotImplementedError("thresholding=True (dynamic thresholding) is not implemented for "
                                      "UniPCMultistepScheduler: it is unsuitable for latent diffusion")
        if solver_p is not None:
            raise NotImplementedError("solver_p (another scheduler as the UniPC predictor) is not implemented")
        if solver_type in ("midpoint", "heun", "logrho"):   # :169-173
            solver_type = "bh1"
        elif solver_type not in ("bh1", "bh2"):
            raise NotImplementedError(f"{solver_type} does is not implemented for {self.__class__}")
        if solver_order not in (1, 2, 3):
            raise ValueError(f"solver_order must be 1, 2 or 3, got {solver_order}")
        if prediction_type not in ("epsilon", "sample", "v_prediction"):
            raise ValueError(f"prediction_type given as {prediction_type} must be one of `epsilon`, `sample`, or"
                             " `v_prediction` for the UniPCMultistepScheduler.")
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                         prediction_type=prediction_type, thresholding=thresholding,
                         dynamic_thresholding_ratio=dynamic_thresholding_ratio, sample_max_value=sample_max_value,
                         predict_x0=predict_x0, solver_type=solver_type, lower_order_final=lower_order_final,
                         disable_corrector=[int(j) for j in disable_corrector], solver_p=None)
        self.predict_x0 = predict_x0
        self.disable_corrector = self.config["disable_corrector"]
        self.model_outputs = [None] * solver_order
        self.timestep_list = [None] * solver_order
        self.lower_order_nums = 0
        self.this_order = None
        self.last_sample = None
        self._rows: dict = {}

    def set_timesteps(self, num_inference_steps: int, device=None):
        """:187-211: DPM-Solver's grid; resets `model_outputs`, `lower_order_nums` and `last_sample`."""
        self._set_grid(num_inference_steps)
        self.model_outputs = [None] * self.config["solver_order"]
        self.lower_order_nums = 0
        self.last_sample = None
        self._orders = self._loop_orders_from(len(self.timesteps), 0)
        self._loop_orders = self._orders
        self._finish_set_timesteps(device)

    def _predictor_order(self, i: int, n: int, lower_order_nums: int) -> int:
        """The UniP order :550-555 picks at step index i of n with `lower_order_nums` earlier steps counted."""
        k = self.config["solver_order"]
        order = min(k, n - i) if self.config["lower_order_final"] else k
        return min(order, lower_order_nums + 1)

    def _loop_orders_from(self, n: int, t_start: int) -> list:
        """(corrector, predictor) orders of a loop over steps t_start..n-1 of an n-step grid. The corrector of step i
        has the order of step i-1's predictor; it is off (0) at the loop's first step, which has no `last_sample`, and
        where i-1 is in `disable_corrector` (:526-528). Entries before t_start are the full loop's."""
        k = self.config["solver_order"]

        def run(start):
            out = []
            for i in range(start, n):
                q = self._predictor_order(i, n, min(i - start, k))
                p = out[-1][1] if i > start and (i - 1) not in self.disable_corrector else 0
                out.append((p, q))
            return out

        return run(0)[:t_start] + run(t_start)

    def order_at(self, i: int) -> tuple:
        """(corrector, predictor) orders of step i in a loop started by `set_timesteps`."""
        return self._orders[i]

    def _uni_terms(self, s0, t, earlier, order: int, corrector: bool):
        """(c_x, c_m, c_b, [r_k], [rho]) of a UniC (`corrector`) or UniP update of `order` from s0 to t, `earlier`
        holding the timesteps of the older history entries, most recent first (:311-379, :415-486, same torch ops in
        the same order)."""
        cfg = self.config
        lambda_t, lambda_s0 = self.lambda_t[t], self.lambda_t[s0]
        alpha_t, alpha_s0 = self.alpha_t[t], self.alpha_t[s0]
        sigma_t, sigma_s0 = self.sigma_t[t], self.sigma_t[s0]
        h = lambda_t - lambda_s0
        rks = [(self.lambda_t[si] - lambda_s0) / h for si in earlier[:order - 1]]
        rk_list = list(rks)
        rks.append(1.0)
        rks = torch.tensor(rks)
        hh = -h if self.predict_x0 else h
        h_phi_1 = torch.expm1(hh)
        h_phi_k = h_phi_1 / hh - 1
        factorial_i = 1
        B_h = hh if cfg["solver_type"] == "bh1" else torch.expm1(hh)
        R, b = [], []
        for i in range(1, order + 1):
            R.append(torch.pow(rks, i - 1))
            b.append(h_phi_k * factorial_i / B_h)
            factorial_i *= i + 1
            h_phi_k = h_phi_k / hh - 1 / factorial_i
        R = torch.stack(R)
        b = torch.tensor(b)
        if corrector:
            rhos = torch.tensor([0.5]) if order == 1 else torch.linalg.solve(R, b)
        else:
            rhos = {1: torch.zeros(0), 2: torch.tensor([0.5])}.get(order)
            if rhos is None:
                rhos = torch.linalg.solve(R[:-1, :-1], b[:-1])
        if self.predict_x0:
            return sigma_t / sigma_s0, alpha_t * h_phi_1, alpha_t * B_h, rk_list, list(rhos)
        return alpha_t / alpha_s0, sigma_t * h_phi_1, sigma_t * B_h, rk_list, list(rhos)

    def _row(self, t: int, t_next: int, before: tuple, p: int, q: int) -> torch.Tensor:
        """The tng_unipc_step row of a step at timestep t towards t_next with corrector order p (0: none) and predictor
        order q; `before`: the timesteps of the steps before, most recent first."""
        key = (t, t_next, before, p, q)
        if key not in self._rows:
            zero = torch.tensor(0.0)
            row = list(self._conversion(t, self.predict_x0)) + [zero] * (NCOEF_UNIPC - 3)
            if p > 0:
                c_x, c_m, c_b, rk, rho = self._uni_terms(before[0], t, before[1:], p, corrector=True)
                row[3:6] = [c_x, c_m, c_b]
                row[6:6 + len(rk)] = rk
                row[8:8 + len(rho) - 1] = rho[:-1]
                row[10] = rho[-1]
            c_x, c_m, c_b, rk, rho = self._uni_terms(t, t_next, before, q, corrector=False)
            row[11:14] = [c_x, c_m, c_b]
            row[14:14 + len(rk)] = rk
            row[16:16 + len(rho)] = rho
            self._rows[key] = torch.stack([torch.as_tensor(c, dtype=torch.float32) for c in row])
        return self._rows[key]

    def _coefficients_at(self, i: int, orders: tuple) -> torch.Tensor:
        tl = self._t_list
        p, q = orders
        before = tuple(tl[i - j] for j in range(1, max(p, q - 1) + 1))
        return self._row(tl[i], 0 if i == len(tl) - 1 else tl[i + 1], before, p, q)

    def _loop_step(self, i: int, model_out, cfg: bool, guidance: float, sample, noise, coef, next_in, bufs, *, B, Cc,
                   HW, split_off):
        """Step i of AudioDiffusion.inference: the converted output goes to slot i mod (k + 1) of k + 1 history slots
        (k = solver_order), so that it never overwrites the m_{i-k} an order-k corrector reads; the corrected sample
        stays in one persistent buffer for the next step's corrector."""
        k = self.config["solver_order"]
        p, q = self._loop_orders[i]
        hist = self._history(bufs, sample, k + 1)
        if "unipc_last" not in bufs.__dict__:
            bufs.unipc_last = torch.zeros(sample.shape, device=sample.device, dtype=torch.float32)
        m_prev = [hist[(i - j) % (k + 1)] for j in range(1, max(p, q - 1) + 1)]
        L.unipc_step(model_out, cfg, guidance, sample, coef[i], p, q, hist[i % (k + 1)], m_prev, bufs.unipc_last,
                     sample, next_in, B=B, Cc=Cc, HW=HW, split_off=split_off)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, return_dict: bool = True, **_unused):
        """:490-572 for NCHW fp32 CUDA tensors: the corrector (when the state allows it), then the predictor of the
        order `lower_order_nums` and `lower_order_final` select; the state is updated as the reference does."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after creating the"
                             " scheduler")
        L.require_cuda(model_output)   # no CPU fallback
        t = int(timestep)
        n = len(self._t_list)
        i = self._t_index.get(t, n - 1)
        k = self.config["solver_order"]
        use_corrector = i > 0 and (i - 1) not in self.disable_corrector and self.last_sample is not None
        p = self.this_order if use_corrector else 0
        q = self._predictor_order(i, n, self.lower_order_nums)
        depth = max(p, q - 1)
        before = tuple(int(s) for s in self.timestep_list[::-1][:depth])
        coef = self._row(t, 0 if i == n - 1 else self._t_list[i + 1], before, p, q).to(sample.device)
        B, Cc, H, W = sample.shape
        m_cur = torch.empty(sample.shape, device=sample.device, dtype=torch.float32)
        m_prev = self.model_outputs[::-1][:depth]
        last = self.last_sample.clone() if p else torch.empty_like(m_cur)
        mo = model_output.float().permute(0, 2, 3, 1).contiguous().view(B * H * W, Cc)   # channels-last rows
        prev = torch.empty_like(m_cur)
        L.unipc_step(mo, False, 1.0, sample.contiguous().float(), coef, p, q, m_cur, m_prev, last, prev, None, B=B,
                     Cc=Cc, HW=H * W)
        self.model_outputs = self.model_outputs[1:] + [m_cur]
        self.timestep_list = self.timestep_list[1:] + [t]
        self.this_order = q
        self.last_sample = last
        if self.lower_order_nums < k:
            self.lower_order_nums += 1
        if not return_dict:
            return (prev,)
        return SchedulerOutput(prev_sample=prev)
