"""Compact stand-ins for reference tensors stored under tests/golden/: a SHA-256 digest for bit-exact comparisons and a
strided sample plus float64 sum for comparisons of large tensors."""
import hashlib

import torch

SAMPLES = 4096


def digest(t):
    """SHA-256 of a contiguous tensor's dtype, shape and bytes."""
    t = t.detach().contiguous()
    h = hashlib.sha256(f"{t.dtype}{list(t.shape)}".encode())
    h.update(t.reshape(-1).view(torch.uint8).numpy().tobytes())
    return h.hexdigest()


def sample(t):
    """Strided sample of a tensor's elements and their float64 sum: what a test compares a full tensor against."""
    flat = t.detach().reshape(-1)
    idx = torch.linspace(0, flat.numel() - 1, min(SAMPLES, flat.numel())).long()
    return {"numel": flat.numel(), "shape": list(t.shape), "idx": idx, "val": flat[idx].clone(), "sum": float(flat.double().sum())}
