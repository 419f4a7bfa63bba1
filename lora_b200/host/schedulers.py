"""Sampling schedulers as per-step coefficient tables (the sampling counterpart of ddpm.py).

diffusers is not installed here; the semantics pinned are those of diffusers 0.11-0.14, the releases
the reference samples with (`EulerAncestralDiscreteScheduler` in its notebooks and `visualize_progress`,
`DDIMScheduler` with Stable Diffusion's scheduler config). Both use the training schedule: 1000
scaled-linear betas 0.00085 -> 0.012, `alphas_cumprod` computed in float32 by torch.

With classifier-free guidance folded in, one sampling step of either scheduler, for either prediction
type, is one linear update

    m_hat   = m_u + g * (m_c - m_u)                  (m: the UNet's output, epsilon or v)
    x_{i+1} = alpha_i * x_i + beta_i * m_hat + gamma_i * z_i
    the UNet's next input is s_{i+1} * x_{i+1} at timestep t_{i+1}

and sampling starts from x_0 = init_noise_sigma * z_0, the UNet's first input s_0 * x_0 at t_0.
`coefficients()` evaluates (alpha, beta, gamma, s_next, t_next) per step in float64 from the
scheduler's float32 tables (sigmas / alphas_cumprod, stored as diffusers stores them);
`pack_table()` rounds them to the float32 table lb_sample_step reads.

Euler-ancestral (EulerAncestralDiscreteScheduler):
  timesteps     linspace(0, 999, N) reversed, as floats
  sigmas        ((1 - acp) / acp) ** 0.5 (float32), np.interp at the timesteps, then [.., 0.0], as float32
  init_noise_sigma = max(sigmas);  scale_model_input(x, t_i) = x / (sigma_i ** 2 + 1) ** 0.5
  step i        epsilon: x0 = x - sigma_i m;  v_prediction: x0 = m (-sigma_i / (sigma_i^2 + 1)^0.5) + x / (sigma_i^2 + 1)
                sigma_up = (sigma_{i+1}^2 (sigma_i^2 - sigma_{i+1}^2) / sigma_i^2) ** 0.5
                sigma_down = (sigma_{i+1}^2 - sigma_up^2) ** 0.5
                x' = x + (x - x0) / sigma_i * (sigma_down - sigma_i) + z * sigma_up
DDIM with eta = 0 (DDIMScheduler, Stable Diffusion's config: steps_offset=1, set_alpha_to_one=False,
clip_sample=False, "leading" spacing):
  timesteps     arange(N) * (1000 // N) reversed, plus 1;  init_noise_sigma = 1; scale_model_input = identity
  step i        prev_t = t_i - 1000 // N;  a = acp[t_i], a_prev = acp[prev_t] if prev_t >= 0 else acp[0]
                epsilon: x0 = (x - (1 - a)^0.5 m) / a^0.5,  eps = m
                v_prediction: x0 = a^0.5 x - (1 - a)^0.5 m,  eps = a^0.5 m + (1 - a)^0.5 x
                x' = a_prev^0.5 x0 + (1 - a_prev)^0.5 eps            (gamma = 0, s = 1)

DDPM / PNDM sampling are not provided: DDPM's strided-variance rule changed between diffusers
releases, and no copy of them is installed to pin it against.
"""
import math

import numpy as np
import torch

SCHEDULERS = ("euler_ancestral", "ddim")
PREDICTION_TYPES = ("epsilon", "v_prediction")
NUM_TRAIN_TIMESTEPS = 1000
TABLE_COLS = 8          # row 0: (init_noise_sigma, s_0, t_0, 0...); row 1 + i: (alpha, beta, gamma, s_next, t_next, last, 0, 0)


def check(scheduler: str, prediction_type: str):
    if scheduler not in SCHEDULERS:
        raise ValueError(f"unknown scheduler {scheduler!r}: one of {SCHEDULERS}")
    if prediction_type not in PREDICTION_TYPES:
        raise ValueError(f"unknown prediction type {prediction_type!r}: one of {PREDICTION_TYPES}")


def alphas_cumprod() -> torch.Tensor:
    """diffusers' scaled_linear schedule, float32 (the same as ddpm.DDPMNoiser's)."""
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, NUM_TRAIN_TIMESTEPS, dtype=torch.float32) ** 2
    return torch.cumprod(1.0 - betas, dim=0)


def timesteps(scheduler: str, n: int) -> np.ndarray:
    """The scheduler's timesteps for n inference steps (float64 for Euler-ancestral, int64 for DDIM)."""
    if scheduler == "euler_ancestral":
        return np.linspace(0, NUM_TRAIN_TIMESTEPS - 1, n, dtype=float)[::-1].copy()
    ratio = NUM_TRAIN_TIMESTEPS // n
    return (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.int64) + 1


def euler_sigmas(n: int) -> np.ndarray:
    """EulerAncestralDiscreteScheduler.sigmas after set_timesteps(n): float32, n + 1 values."""
    acp = alphas_cumprod()
    base = np.array(((1 - acp) / acp) ** 0.5)
    s = np.interp(timesteps("euler_ancestral", n), np.arange(0, len(base)), base)
    return np.concatenate([s, [0.0]]).astype(np.float32)


def init_noise_sigma(scheduler: str, n: int) -> float:
    return float(euler_sigmas(n).max()) if scheduler == "euler_ancestral" else 1.0


def coefficients(scheduler: str, prediction_type: str, n: int):
    """((init_noise_sigma, s_0, t_0), steps): steps is a float64 [n, 5] array of
    (alpha, beta, gamma, s_next, t_next) per step, evaluated in float64."""
    check(scheduler, prediction_type)
    if n < 1:
        raise ValueError(f"num_inference_steps must be at least 1, got {n}")
    ts = timesteps(scheduler, n).astype(np.float64)
    steps = np.zeros((n, 5), dtype=np.float64)
    v = prediction_type == "v_prediction"
    if scheduler == "euler_ancestral":
        sig = euler_sigmas(n).astype(np.float64)
        for i in range(n):
            s, s_to = sig[i], sig[i + 1]
            up = math.sqrt(s_to ** 2 * (s ** 2 - s_to ** 2) / s ** 2)
            down = math.sqrt(s_to ** 2 - up ** 2)
            d = down - s
            if v:
                alpha, beta = 1.0 + d * s / (s ** 2 + 1), d / math.sqrt(s ** 2 + 1)
            else:
                alpha, beta = 1.0, d
            steps[i] = (alpha, beta, up, 1.0 / math.sqrt(s_to ** 2 + 1), ts[i + 1] if i + 1 < n else 0.0)
        return (float(sig.max()), 1.0 / math.sqrt(sig[0] ** 2 + 1), ts[0]), steps
    acp = alphas_cumprod().double().numpy()
    ratio = NUM_TRAIN_TIMESTEPS // n
    for i in range(n):
        t = int(ts[i])
        a = acp[t]
        prev = t - ratio
        ap = acp[prev] if prev >= 0 else acp[0]
        sa, sb, sap, sbp = math.sqrt(a), math.sqrt(1 - a), math.sqrt(ap), math.sqrt(1 - ap)
        if v:
            alpha, beta = sap * sa + sbp * sb, sbp * sa - sap * sb
        else:
            alpha, beta = sap / sa, sbp - sap * sb / sa
        steps[i] = (alpha, beta, 0.0, 1.0, ts[i + 1] if i + 1 < n else 0.0)
    return (1.0, 1.0, ts[0]), steps


def pack_table(scheduler: str, prediction_type: str, n: int, max_steps: int) -> torch.Tensor:
    """The float32 [max_steps + 1, TABLE_COLS] table lb_sample_step reads (rows past n are zero)."""
    if n > max_steps:
        raise ValueError(f"num_inference_steps {n} exceeds max_steps {max_steps}")
    (sigma0, s0, t0), steps = coefficients(scheduler, prediction_type, n)
    tab = np.zeros((max_steps + 1, TABLE_COLS), dtype=np.float64)
    tab[0, :3] = (sigma0, s0, t0)
    tab[1:n + 1, :5] = steps
    tab[n, 5] = 1.0
    return torch.from_numpy(tab.astype(np.float32))
