"""ORACLE (test infrastructure only): the reference's training step with the scheduler's
`prediction_type` (lora_diffusion/cli_lora_pti.py:333-338, train_lora_dreambooth.py:846-853):

    "epsilon"       target = noise
    "v_prediction"  target = scheduler.get_velocity(latents, noise, timesteps)
    anything else   ValueError(f"Unknown prediction type {prediction_type}")

`get_velocity` is restated from the noiser's tables (diffusers' DDPMScheduler.get_velocity:
sqrt(acp[t]) * noise - sqrt(1 - acp[t]) * sample). Everything else -- noising, mask, prior
preservation, inpainting input, optimizer -- is oracle/ref_step.py's and oracle/joint_ref.py's, unchanged:
the target is the only thing the prediction type changes, and those steps use `noise` only to noise
the latents and as the target, so the velocity is passed in its place with the noised latents fixed
beforehand.

Pinned: `forward_loss(prediction_type="v_prediction")` reproduces the reference's own `loss_step`
run with a v-prediction scheduler to 2e-6 relative (plain, t_mutliplier, masked, inpainting, and
the tiny SD2 models) -- tests/golden/pti_loss_step_v.pt, written by
scripts/make_golden.py::gen_loss_step_v, checked in tests/test_sd2_cpu.py. Imports nothing from the
product package.
"""
from .joint_ref import RefJointStep
from .ref_step import RefDreamboothStep

PREDICTION_TYPES = ("epsilon", "v_prediction")


def get_velocity(noiser, latents, noise, timesteps):
    a = noiser.sqrt_acp[timesteps].view(-1, 1, 1, 1).to(latents.dtype)
    s = noiser.sqrt_one_minus_acp[timesteps].view(-1, 1, 1, 1).to(latents.dtype)
    return a * noise - s * latents


class _Noised:
    """Stands in for the noiser inside one forward_loss call: add_noise returns the latents noised
    with the real noise, whatever `noise` argument the loss receives (the velocity)."""

    def __init__(self, noiser, noisy):
        self._noiser, self._noisy = noiser, noisy

    def add_noise(self, latents, noise, timesteps):
        return self._noisy

    def __getattr__(self, name):
        return getattr(self._noiser, name)


class PredictionTypeLoss:
    """forward_loss with a `prediction_type` keyword; mixed in before a step class of this package."""

    def forward_loss(self, latents, input_ids, noise, timesteps, prediction_type="epsilon", **loss_kw):
        if prediction_type not in PREDICTION_TYPES:
            raise ValueError(f"Unknown prediction type {prediction_type}")
        if prediction_type == "epsilon":
            return super().forward_loss(latents, input_ids, noise, timesteps, **loss_kw)
        noiser = self.noiser
        target = get_velocity(noiser, latents, noise, timesteps)
        self.noiser = _Noised(noiser, noiser.add_noise(latents, noise, timesteps))
        try:
            return super().forward_loss(latents, input_ids, target, timesteps, **loss_kw)
        finally:
            self.noiser = noiser


class RefDreamboothStepV(PredictionTypeLoss, RefDreamboothStep):
    """oracle/ref_step.py's step; `step(..., prediction_type=...)` passes it on to forward_loss."""


class RefJointStepV(PredictionTypeLoss, RefJointStep):
    """oracle/joint_ref.py's LoRA + embedding-table step with the prediction type."""
