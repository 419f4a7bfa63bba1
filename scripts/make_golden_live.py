"""Run the parity scenarios of tests/test_vs_reference_live.py and tests/test_formats_cpu.py against
the reference project (cloneofsimo/lora, a checkout given by path) and store what it returned:

    python scripts/make_golden_live.py /path/to/lora

  tests/golden/reference_live.json   digests (oracle/fingerprint.py) of what each scenario returned
  tests/golden/reference_modules.pt  the reference operator classes' outputs and gradients

The reference package import needs fire / diffusers, which the functions under test never call:
its files are loaded by path into a stub package with empty stand-ins for both."""
import importlib.util
import json
import os
import sys
import tempfile
import types
from pathlib import Path

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.fingerprint import digest, fingerprint  # noqa: E402


def load_ref(ref_dir, fname, modname):
    for stub, attrs in {"fire": {"Fire": lambda *a, **k: None},
                        "diffusers": {"StableDiffusionPipeline": object}}.items():
        if stub not in sys.modules:
            m = types.ModuleType(stub)
            for k, v in attrs.items():
                setattr(m, k, v)
            sys.modules[stub] = m
    if "lora_diffusion_ref" not in sys.modules:
        pkg = types.ModuleType("lora_diffusion_ref")
        pkg.__path__ = [ref_dir]
        sys.modules["lora_diffusion_ref"] = pkg
    full = f"lora_diffusion_ref.{modname}"
    if full not in sys.modules:
        spec = importlib.util.spec_from_file_location(full, os.path.join(ref_dir, fname))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[full] = mod
        spec.loader.exec_module(mod)
    return sys.modules[full]


def main(ref_root):
    ref_dir = os.path.join(ref_root, "lora_diffusion")
    R = load_ref(ref_dir, "lora.py", "lora")
    manager = load_ref(ref_dir, "lora_manager.py", "lora_manager")
    ckpt = load_ref(ref_dir, "to_ckpt_v2.py", "to_ckpt_v2")
    adder = load_ref(ref_dir, "cli_lora_add.py", "cli_lora_add")
    import test_formats_cpu as F
    import test_vs_reference_live as V

    out = {"public_names": V.public_names(R), "signatures": fingerprint(V.signatures(R))}
    per_key = lambda d: {k: digest(v) for k, v in d.items()}
    with tempfile.TemporaryDirectory() as d:
        out["inject_save_load"] = per_key(V.inject_save_load(R, Path(d)))
    out["inject_order"] = digest(V.inject_order(R))
    with tempfile.TemporaryDirectory() as d:
        out["small_helpers"] = per_key(V.small_helpers(R, Path(d)))
    with tempfile.TemporaryDirectory() as d:
        j = F.join_case(manager, Path(d))
        out["join"] = {"ranklist": j["ranklist"], "toks": j["toks"],
                       **{k: digest(j[k]) for k in ("meta", "keys", "tensors")}}
    with tempfile.TemporaryDirectory() as d:
        out["add"] = {m: {k: digest(v) for k, v in c.items()} for m, c in F.add_case(adder, Path(d)).items()}
    out["ckpt"] = per_key(F.ckpt_case(ckpt))
    gold = os.path.join(ROOT, "tests", "golden")
    with open(os.path.join(gold, "reference_live.json"), "w") as fh:
        json.dump(out, fh, separators=(",", ":"))
    torch.save(V.reference_module_outputs(R), os.path.join(gold, "reference_modules.pt"))


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
