"""Stored outputs of the unmodified reference (tests/golden/ref_compare.pt.gz, written by tests/golden/make_goldens_ref_compare.py).

Host-side data structures that must match the reference bit for bit (loader windows, signal snapshots) are stored as digests of
(dtype, shape, bytes): equal digests mean equal tensors, at a fraction of the file size."""
import gzip
import hashlib
import os

import torch

PATH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ref_compare.pt.gz")


def digest(t):
    """None, or (dtype, shape, sha256 of the contiguous bytes) of a tensor."""
    if t is None:
        return None
    t = t.detach().contiguous().cpu()
    return (str(t.dtype), tuple(t.shape), hashlib.sha256(t.view(torch.uint8).numpy().tobytes() if t.numel() else b"").hexdigest())


_cache = None


def load():
    global _cache
    if _cache is None:
        with gzip.open(PATH, "rb") as f:
            _cache = torch.load(f, weights_only=False)
    return _cache
