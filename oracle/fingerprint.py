"""JSON-able fingerprints of what a reference run returned, for tests that compare with stored
results of the original project (scripts/make_golden_live.py writes them, tests/golden/ keeps them).

Tensors become (dtype, shape, sha256 of the raw bytes), so equal fingerprints mean bitwise-equal
tensors -- the same check as torch.equal on the live objects; containers and scalars keep their
structure. Sets are sorted, tuples become lists. digest() condenses a fingerprint to one hash."""
import hashlib
import json

import torch


def fingerprint(x):
    if isinstance(x, torch.Tensor):
        t = x.detach().cpu().contiguous()
        raw = t.reshape(-1).view(torch.uint8).numpy().tobytes() if t.numel() else b""
        return ["tensor", str(t.dtype), list(t.shape), hashlib.sha256(raw).hexdigest()]
    if isinstance(x, dict):
        return {str(k): fingerprint(v) for k, v in x.items()}
    if isinstance(x, (set, frozenset)):
        return sorted(fingerprint(v) for v in x)
    if isinstance(x, (list, tuple)):
        return [fingerprint(v) for v in x]
    if isinstance(x, bytes):
        return ["bytes", hashlib.sha256(x).hexdigest()]
    if x is None or isinstance(x, (str, int, float, bool)):
        return x
    return repr(x)


def digest(x):
    return hashlib.sha256(json.dumps(fingerprint(x), sort_keys=True).encode()).hexdigest()
