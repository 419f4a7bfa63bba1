"""Rank-concatenation of LoRA files ("join") and the small manager object that drives a joined
model -- the host-side file arithmetic next to `collapse_lora`.

Behaviour follows the reference's `lora_diffusion/lora_manager.py` (`lora_join` :13-71,
`DummySafeTensorObject` :74-86, `LoRAManager` :89-144); tests/test_formats_cpu.py runs both side
by side on the same files.

Algebra: for LoRAs (B_i [N, r_i], A_i [r_i, K]) the matrices B = [B_1 | B_2 | ...] and
A = [A_1 ; A_2 ; ...] satisfy B.A = sum_i B_i.A_i, so a join is one LoRA of rank sum r_i. A
per-source strength s_i is then the diagonal (s_1 x r_1, s_2 x r_2, ...) between the factors --
`set_lora_diag`, which the fused kernels take as their `diag` argument. The kernels keep the rank
axis in 16 operand rows: a joined rank above 16 raises `LoraB200Error` at the first forward;
joining itself is file-level and unlimited.
"""
from dataclasses import dataclass, field
from typing import Dict, List

import torch

EMBED = "<embed>"                      # metadata value that marks a key as a learned token embedding
_MODEL_PREFIXES = ("text_encoder", "unet")


def _declared_rank(meta: Dict[str, str]) -> int:
    seen = {int(value) for key, value in meta.items() if key.endswith("rank")}
    assert len(seen) <= 1, "Rank should be the same per model"
    return seen.pop() if seen else 0


@dataclass
class _Join:
    """Accumulates the joined tensors / metadata of a list of safetensors-like handles."""
    tensors: Dict[str, torch.Tensor] = field(default_factory=dict)
    metadata: Dict[str, str] = field(default_factory=dict)
    ranks: List[int] = field(default_factory=list)
    tokens_per_file: List[int] = field(default_factory=list)

    def add_metadata(self, metas):
        pooled = {}
        for m in metas:
            self.ranks.append(_declared_rank(m))
            pooled.update(m)
        # token entries are re-issued under new names by add_tokens()
        self.metadata.update((k, v) for k, v in pooled.items() if v != EMBED)

    def add_factors(self, handles):
        width = sum(self.ranks)
        names = set().union(*(set(h.keys()) for h in handles))
        for name in names:
            if not name.startswith(_MODEL_PREFIXES):
                continue
            rank_axis = 0 if name.endswith("down") else 1          # A: [r, K]   B: [N, r]
            wide = torch.cat([h.get_tensor(name) for h in handles], dim=rank_axis)
            assert wide.shape[rank_axis] == width
            self.tensors[name] = wide
            self.metadata[name[: name.rindex(":")] + ":rank"] = str(width)

    def add_tokens(self, handles):
        for file_no, h in enumerate(handles):
            own = sorted(key for key, value in h.metadata().items() if value == EMBED)
            for slot, old in enumerate(own):
                fresh = f"<s{file_no}-{slot}>"
                self.tensors[fresh] = h.get_tensor(old)
                self.metadata[fresh] = EMBED
                print(f"Embedding {old} replaced to {fresh}")
            self.tokens_per_file.append(len(own))


def lora_join(lora_safetenors: list):
    """(tensors, metadata, ranklist, token_size_list) of the join of the given handles (anything
    with `.keys()`, `.metadata()`, `.get_tensor()`); the argument keeps the reference's spelling."""
    j = _Join()
    j.add_metadata([dict(h.metadata()) for h in lora_safetenors])
    j.add_factors(lora_safetenors)
    j.add_tokens(lora_safetenors)
    return j.tensors, j.metadata, j.ranks, j.tokens_per_file


class DummySafeTensorObject:
    """Dict-backed object with the three read calls of a `safe_open` handle."""

    def __init__(self, tensor: dict, metadata):
        self.tensor, self._metadata = tensor, metadata

    def keys(self):
        return self.tensor.keys()

    def metadata(self):
        return self._metadata

    def get_tensor(self, key):
        return self.tensor[key]


class LoRAManager:
    """Patches the join of several LoRA files into `pipe` (anything with `.unet`,
    `.text_encoder`, `.tokenizer`). `tune([s_1, ...])`: one strength per file; `prompt(text)`:
    `<k>` (1-based) becomes file k's embedding tokens."""

    def __init__(self, lora_paths_list: List[str], pipe):
        self.lora_paths_list, self.pipe = lora_paths_list, pipe
        self._setup()

    def _setup(self):
        from safetensors import safe_open
        from .patch import apply_learned_embed_in_clip, monkeypatch_or_replace_safeloras
        from .persist import parse_safeloras_embeds
        self._lora_safetenors = [safe_open(path, framework="pt", device="cpu") for path in self.lora_paths_list]
        tensors, meta, self.ranklist, self.token_size_list = lora_join(self._lora_safetenors)
        self.total_safelora = DummySafeTensorObject(tensors, meta)
        monkeypatch_or_replace_safeloras(self.pipe, self.total_safelora)
        apply_learned_embed_in_clip(parse_safeloras_embeds(self.total_safelora), self.pipe.text_encoder,
                                    self.pipe.tokenizer, token=None, idempotent=True)

    def tune(self, scales):
        from .patch import set_lora_diag
        assert len(scales) == len(self.ranklist), "Scale list should be the same length as ranklist"
        per_rank = torch.repeat_interleave(torch.as_tensor(scales, dtype=torch.float32),
                                           torch.as_tensor(self.ranklist))
        set_lora_diag(self.pipe.unet, per_rank)

    def diag_rows(self, per_image_scales) -> torch.Tensor:
        """The selector diagonals `tune()` would set, one row per image: per_image_scales is B lists of
        one strength per file; returns [B, total_rank] fp32, for `per_sample_lora(diag=...)` or the
        samplers' `lora_diag={"unet": ...}` (every image of one batch with its own mix)."""
        rows = []
        for scales in per_image_scales:
            assert len(scales) == len(self.ranklist), "Scale list should be the same length as ranklist"
            rows.append(torch.repeat_interleave(torch.as_tensor(scales, dtype=torch.float32),
                                                torch.as_tensor(self.ranklist)))
        return torch.stack(rows)

    def prompt(self, prompt):
        if prompt is None:
            return prompt
        for file_no, count in enumerate(self.token_size_list):
            prompt = prompt.replace(f"<{file_no + 1}>", "".join(f"<s{file_no}-{k}>" for k in range(count)))
        return prompt
