"""CPU restatement of text-guided editing and inpainting (TEST INFRASTRUCTURE ONLY).

Follows the vendored diffusers fork's StableDiffusionImg2ImgPipeline (pipeline_stable_diffusion_img2img.py:509-570)
and StableDiffusionInpaintPipelineLegacy (pipeline_stable_diffusion_inpaint_legacy.py:514-528, 640-709) on top of
oracle/pipeline.py's denoising loop; img2img is the legacy-inpaint loop without a mask. The audio side is AudioLDM's:
latents are `scale_factor * posterior.sample()` (audioldm/variational_autoencoder/autoencoder.py:126-135) and ratio
masks follow audioldm/ldm.py:773-777. Randomness is injected: `eps_post` (posterior), `noise` (add-noise draw) and
`step_noises[k]` (the DDPM draw of the k-th executed step); `seeded_draws` regenerates them from a case's seed.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch

from . import unet as ounet


def input_wave(n_samples: int, seed: int) -> torch.Tensor:
    """The seeded 16 kHz input clip of the edit goldens: two tones, one of them gliding, plus seeded noise."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n_samples, dtype=torch.float64) / 16000.0
    w = 0.4 * torch.sin(2 * math.pi * 440.0 * t) + 0.2 * torch.sin(2 * math.pi * 1234.5 * t * (1 + t))
    return (w.float() + 0.05 * torch.randn(n_samples, generator=g)).contiguous()


def seeded_draws(seed: int, shape, n_step_draws: int):
    """The fork pipelines' draws from a CPU generator seeded with `seed`, in their order: the posterior noise, the
    add-noise draw, then one draw per executed DDPM step with t > 0 (randn_tensor on the CPU is torch.randn)."""
    g = torch.Generator().manual_seed(seed)
    eps_post = torch.randn(shape, generator=g)
    noise = torch.randn(shape, generator=g)
    return eps_post, noise, [torch.randn(shape, generator=g) for _ in range(n_step_draws)]


def get_timesteps(num_steps: int, strength: float) -> int:
    """img2img :509-516: the index t_start of the first executed timestep."""
    init_timestep = min(int(num_steps * strength), num_steps)
    return max(num_steps - init_timestep, 0)


def add_noise(alphas_cumprod: torch.Tensor, x0: torch.Tensor, noise: torch.Tensor, t) -> torch.Tensor:
    """scheduling_ddpm.py:351-372 for one timestep (fp32 `** 0.5`, broadcast over the batch)."""
    a = alphas_cumprod[torch.tensor([int(t)])]
    return (a ** 0.5).reshape(-1, 1, 1, 1) * x0 + ((1 - a) ** 0.5).reshape(-1, 1, 1, 1) * noise


def latents_from_moments(moments: torch.Tensor, eps_post: torch.Tensor, scale_factor: float) -> torch.Tensor:
    """DiagonalGaussianDistribution(moments).sample() with the draw `eps_post`, times scale_factor."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    std = torch.exp(0.5 * torch.clamp(logvar, -30.0, 20.0))
    return scale_factor * (mean + std * eps_post)


def ratio_mask(H: int, W: int, time_ratio=None, freq_ratio=None) -> torch.Tensor:
    """ldm.py:773-777 at latent resolution: ones, time rows / mel-bin columns of the bands zeroed. (1, 1, H, W)."""
    t0, t1 = time_ratio if time_ratio is not None else (1.0, 1.0)
    f0, f1 = freq_ratio if freq_ratio is not None else (1.0, 1.0)
    m = torch.ones(1, H, W)
    m[:, int(H * t0):int(H * t1), :] = 0
    m[:, :, int(W * f0):int(W * f1)] = 0
    return m[:, None]


def edit_loop(unet_sd, unet_cfg, scheduler, prompt_embeds, mask, num_steps, guidance_scale, strength, x0, noise,
              step_noises: Optional[List[torch.Tensor]] = None, inpaint_mask: Optional[torch.Tensor] = None,
              trace: Optional[list] = None) -> torch.Tensor:
    """inpaint_legacy:640-709 (add_predicted_noise=False); with `inpaint_mask` None it is img2img's loop."""
    cfg = guidance_scale > 1.0
    scheduler.set_timesteps(num_steps)
    t_start = get_timesteps(num_steps, strength)
    timesteps = scheduler.timesteps[t_start:]
    ac = scheduler.alphas_cumprod
    latents = add_noise(ac, x0, noise, timesteps[0])
    for k, t in enumerate(timesteps):
        x = torch.cat([latents] * 2) if cfg else latents
        pred = ounet.unet_forward(unet_sd, unet_cfg, x, t, prompt_embeds, mask)
        if cfg:
            u, c = pred.chunk(2)
            pred = u + guidance_scale * (c - u)
        if step_noises is not None:
            latents = scheduler.step(pred, t, latents, step_noises[k] if int(t) > 0 else None)
        else:
            latents = scheduler.step(pred, t, latents)
        if inpaint_mask is not None:
            latents = (add_noise(ac, x0, noise, t) * inpaint_mask) + (latents * (1 - inpaint_mask))
        if trace is not None:
            trace.append(latents.clone())
    if inpaint_mask is not None:
        latents = (x0 * inpaint_mask) + (latents * (1 - inpaint_mask))
    return latents
