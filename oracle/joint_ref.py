"""ORACLE (test infrastructure only): the reference's two loops that train the LoRA factors and the
CLIP token-embedding table in ONE torch.optim.AdamW, in plain PyTorch eager.

mode="table"  lora_diffusion/cli_lora_pti.py phase 2 with `continue_inversion` (:958-997 builds
    the optimizer, :545-620 is `perform_tuning`): param groups [unet LoRA, embedding table,
    text LoRA if any], AdamW(weight_decay=weight_decay_lora) over the dense table; per iteration
    lr_scheduler.step() FIRST, zero_grad, loss_step, backward,
    clip_grad_norm_(unet.parameters() + text_encoder.parameters()), optimizer.step(). Nothing is
    restored. Pinned: 3 iterations of the reference's real `perform_tuning` built that way
    (tests/golden/pti_continue_inversion.pt, scripts/make_golden.py::gen_continue_inversion):
    per-step loss to 5e-6 relative and the whole table after every step to 2e-7.

mode="placeholders"  training_scripts/train_lora_w_ti.py (:830-853 builds the optimizer,
    :986-1075 is the loop): param groups [unet LoRA, text LoRA, table]; at iteration k the LoRA
    groups get lr 0 while k < unfreeze_lora_step, else their base lr and the table 0; loss, backward,
    clip_grad_norm_ over UNet + text encoder, optimizer.step(), lr_scheduler.step(), zero_grad, then
    every table row except the placeholders is restored from the original table. That loop lives
    inside the script's main() and cannot be called, so this is a line-by-line restatement of
    :986-1075 with no golden of its own (its loss, clip and AdamW are the pieces pinned above).

Built on oracle/ref_step.py (loss) and oracle/ref_modules.py (LoRA sites); imports nothing from
the product package.
"""
import itertools
import warnings
from typing import Callable, List, Optional, Sequence

import torch

from .ref_step import RefDreamboothStep


class RefJointStep(RefDreamboothStep):
    def __init__(self, unet, text_encoder, noiser, unet_sites: List, text_sites: Optional[List], mode: str,
                 lr: float, lr_text: float, lr_embedding: float, lr_lambda: Callable[[int], float],
                 weight_decay: float, betas=(0.9, 0.999), eps=1e-8, max_grad_norm=1.0,
                 t_multiplier: float = 1.0, autocast_dtype=None,
                 placeholder_token_ids: Sequence[int] = (), unfreeze_lora_step: int = 500):
        if mode not in ("table", "placeholders"):
            raise ValueError(mode)
        super().__init__(unet, text_encoder, noiser, unet_sites, text_sites, lr=lr, lr_text=lr_text, betas=betas,
                         weight_decay=weight_decay, eps=eps, max_grad_norm=max_grad_norm,
                         t_multiplier=t_multiplier, autocast_dtype=autocast_dtype)
        self.mode = mode
        self.lr, self.lr_text = lr, lr_text
        self.unfreeze_lora_step = unfreeze_lora_step
        self.train_text = True                 # the text encoder runs with gradients (the table trains)
        emb = text_encoder.get_input_embeddings()
        emb.weight.requires_grad_(True)
        self.table = emb.weight
        self.orig = emb.weight.detach().clone()
        unet_g = {"params": self.unet_params, "lr": lr}
        table_g = {"params": [emb.weight], "lr": lr_embedding}
        text_g = {"params": self.text_params, "lr": lr_text}
        if mode == "table":                     # cli_lora_pti.py:958-993
            groups = [unet_g, table_g] + ([text_g] if self.text_params else [])
        else:                                   # train_lora_w_ti.py:830-840
            if not self.text_params:
                raise ValueError("mode='placeholders' needs text-encoder LoRA sites")
            groups = [unet_g, text_g, table_g]
        self.opt = torch.optim.AdamW(groups, lr=lr, betas=betas, weight_decay=weight_decay, eps=eps)
        self.sched = torch.optim.lr_scheduler.LambdaLR(self.opt, lr_lambda)
        keep = torch.zeros(self.orig.shape[0], dtype=torch.bool, device=self.orig.device)
        keep[list(placeholder_token_ids)] = True
        self.index_no_updates = ~keep
        self.k = 0

    def lrs(self) -> List[float]:
        return [g["lr"] for g in self.opt.param_groups]

    def _clip(self):
        if self.max_grad_norm:
            torch.nn.utils.clip_grad_norm_(itertools.chain(self.unet.parameters(), self.text_encoder.parameters()),
                                           self.max_grad_norm)

    def step(self, latents, input_ids, noise=None, timesteps=None, **loss_kw):
        if noise is None:
            noise = torch.randn_like(latents)
        if timesteps is None:
            t_max = int(self.noiser.num_train_timesteps * self.t_multiplier)
            timesteps = torch.randint(0, t_max, (latents.shape[0],), device=latents.device).long()
        with warnings.catch_warnings():        # the PTI order steps the scheduler before the optimizer
            warnings.simplefilter("ignore", UserWarning)
            if self.mode == "table":
                self.sched.step()                                           # :587
                self.opt.zero_grad()                                        # :589
                loss = self.forward_loss(latents, input_ids, noise, timesteps, **loss_kw)
                loss.backward()
                self._clip()                                                # :606-608
                self.opt.step()                                             # :609
            else:
                g = self.opt.param_groups
                if self.k < self.unfreeze_lora_step:                        # :988-991
                    g[0]["lr"] = 0.0
                    g[1]["lr"] = 0.0
                else:                                                       # :992-995
                    g[0]["lr"] = self.lr
                    g[1]["lr"] = self.lr_text
                    g[2]["lr"] = 0.0
                loss = self.forward_loss(latents, input_ids, noise, timesteps, **loss_kw)
                loss.backward()
                self._clip()                                                # :1057-1063
                self.opt.step()                                             # :1065
                self.sched.step()                                           # :1066
                self.opt.zero_grad()                                        # :1068
                with torch.no_grad():                                       # :1070-1075
                    self.table[self.index_no_updates] = self.orig[self.index_no_updates]
        self.k += 1
        return loss.detach()
