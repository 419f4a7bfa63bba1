"""ORACLE (test infrastructure only -- never imported by the product path).

diffusers' DPMSolverMultistepScheduler (releases 0.11-0.14) in its DPM-Solver++(2M) form, written op by op
as the scheduler writes it: float32 alpha_t / sigma_t / lambda_t tables, convert_model_output, the
`model_outputs` list and `lower_order_nums`, the first- and second-order (midpoint) updates, and
add_noise. No diffusers copy is installed to run against: this restates the source of those releases.
It plugs into the loops of oracle/sample_ref.py (`sample`) and oracle/sample_image_ref.py
(`sample_img2img`, `sample_inpaint`) like their own schedulers. Run it in float64 or in the run's dtype.
"""
import numpy as np
import torch

from . import sample_ref as R


class RefDPMSolverMultistep:
    """DPMSolverMultistepScheduler (scaled_linear, 1000 steps) with solver_order=2,
    algorithm_type="dpmsolver++", solver_type="midpoint", lower_order_final=True, thresholding=False.
    `step` takes the step's index, as sample_ref's schedulers do, where the scheduler looks the index up
    from the timestep (the same index: the timesteps are distinct)."""

    def __init__(self, prediction_type="epsilon"):
        self.prediction_type = prediction_type
        self.alphas_cumprod = R._alphas_cumprod()
        self.alpha_t = torch.sqrt(self.alphas_cumprod)
        self.sigma_t = torch.sqrt(1 - self.alphas_cumprod)
        self.lambda_t = torch.log(self.alpha_t) - torch.log(self.sigma_t)
        self.init_noise_sigma = 1.0
        self.solver_order = 2
        self.lower_order_final = True

    def set_timesteps(self, n, device="cpu"):
        ts = np.linspace(0, 999, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        self.timesteps = torch.from_numpy(ts).to(device)
        self.model_outputs = [None] * self.solver_order
        self.lower_order_nums = 0

    def scale_model_input(self, sample, i):
        return sample

    def convert_model_output(self, model_output, timestep, sample):
        alpha_t, sigma_t = self.alpha_t[timestep], self.sigma_t[timestep]
        if self.prediction_type == "epsilon":
            return (sample - sigma_t * model_output) / alpha_t
        return alpha_t * sample - sigma_t * model_output

    def dpm_solver_first_order_update(self, model_output, timestep, prev_timestep, sample):
        lambda_t, lambda_s = self.lambda_t[prev_timestep], self.lambda_t[timestep]
        alpha_t = self.alpha_t[prev_timestep]
        sigma_t, sigma_s = self.sigma_t[prev_timestep], self.sigma_t[timestep]
        h = lambda_t - lambda_s
        return (sigma_t / sigma_s) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * model_output

    def multistep_dpm_solver_second_order_update(self, model_output_list, timestep_list, prev_timestep, sample):
        t, s0, s1 = prev_timestep, timestep_list[-1], timestep_list[-2]
        m0, m1 = model_output_list[-1], model_output_list[-2]
        lambda_t, lambda_s0, lambda_s1 = self.lambda_t[t], self.lambda_t[s0], self.lambda_t[s1]
        alpha_t = self.alpha_t[t]
        sigma_t, sigma_s0 = self.sigma_t[t], self.sigma_t[s0]
        h, h_0 = lambda_t - lambda_s0, lambda_s0 - lambda_s1
        r0 = h_0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1)

    def step(self, model_output, i, sample, noise=None):
        n = len(self.timesteps)
        timestep = int(self.timesteps[i])
        prev_timestep = 0 if i == n - 1 else int(self.timesteps[i + 1])
        lower_order_final = i == n - 1 and self.lower_order_final and n < 15
        model_output = self.convert_model_output(model_output, timestep, sample)
        for k in range(self.solver_order - 1):
            self.model_outputs[k] = self.model_outputs[k + 1]
        self.model_outputs[-1] = model_output
        if self.lower_order_nums < 1 or lower_order_final:
            prev_sample = self.dpm_solver_first_order_update(model_output, timestep, prev_timestep, sample)
        else:
            timestep_list = [int(self.timesteps[i - 1]), timestep]
            prev_sample = self.multistep_dpm_solver_second_order_update(self.model_outputs, timestep_list,
                                                                        prev_timestep, sample)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        return prev_sample

    def add_noise(self, original_samples, noise, timesteps):
        """sqrt(acp[t]) * original + sqrt(1 - acp[t]) * noise, acp cast to the samples' dtype (the same rule
        as DDIM's add_noise)."""
        alphas_cumprod = self.alphas_cumprod.to(device=original_samples.device, dtype=original_samples.dtype)
        timesteps = timesteps.to(original_samples.device)
        sqrt_alpha_prod = (alphas_cumprod[timesteps] ** 0.5).flatten()
        while len(sqrt_alpha_prod.shape) < len(original_samples.shape):
            sqrt_alpha_prod = sqrt_alpha_prod.unsqueeze(-1)
        sqrt_one_minus_alpha_prod = ((1 - alphas_cumprod[timesteps]) ** 0.5).flatten()
        while len(sqrt_one_minus_alpha_prod.shape) < len(original_samples.shape):
            sqrt_one_minus_alpha_prod = sqrt_one_minus_alpha_prod.unsqueeze(-1)
        return sqrt_alpha_prod * original_samples + sqrt_one_minus_alpha_prod * noise
