"""DDPM forward-noising used by the training loops (stands in for diffusers' DDPMScheduler:
scaled-linear betas 0.00085 -> 0.012, 1000 steps; call sites
training_scripts/train_lora_dreambooth.py:678-680,837 and lora_diffusion/cli_lora_pti.py:306).
The schedule is the same for SD 1.x and SD 2.x. The regression target is chosen by the step
(StepConfig.prediction_type): the noise itself for "epsilon", `get_velocity` for "v_prediction"
(SD 2.x 768-v; cli_lora_pti.py:333-338)."""
import torch


class DDPMNoiser:
    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085,
                 beta_end: float = 0.012, device="cpu"):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps,
                               dtype=torch.float32) ** 2
        acp = torch.cumprod(1.0 - betas, dim=0)
        self.num_train_timesteps = num_train_timesteps
        self.sqrt_acp = acp.sqrt().to(device)
        self.sqrt_one_minus_acp = (1.0 - acp).sqrt().to(device)

    def to(self, device):
        self.sqrt_acp = self.sqrt_acp.to(device)
        self.sqrt_one_minus_acp = self.sqrt_one_minus_acp.to(device)
        return self

    def add_noise(self, x0: torch.Tensor, noise: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        a = self.sqrt_acp[t].view(-1, 1, 1, 1).to(x0.dtype)
        b = self.sqrt_one_minus_acp[t].view(-1, 1, 1, 1).to(x0.dtype)
        return a * x0 + b * noise

    def get_velocity(self, x0: torch.Tensor, noise: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """diffusers' DDPMScheduler.get_velocity: sqrt_acp[t] * noise - sqrt_one_minus_acp[t] * x0."""
        a = self.sqrt_acp[t].view(-1, 1, 1, 1).to(x0.dtype)
        b = self.sqrt_one_minus_acp[t].view(-1, 1, 1, 1).to(x0.dtype)
        return a * noise - b * x0
