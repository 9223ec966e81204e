"""Seeded inputs of the paired-metric tests (tests/golden/make_metrics_golden.py, test_metrics_cpu.py, test_metrics_gpu.py).

Images and synthetic LPIPS weights are regenerated from their seeds with uniform draws, box filters and clipping only
(no transcendental functions, so every host makes the same bytes); the golden pins them by SHA-256.  Frames are
[N,3,H,W] float32 in [0,1], the metric classes' input.
"""
import hashlib

import numpy as np
import torch
from scipy.ndimage import uniform_filter

# name -> (n, size, kind, seed)
CASES = {
    "rand256": (3, 256, "noisy", 11),
    "rand512": (1, 512, "noisy", 12),
    "nonneg": (2, 64, "nonneg", 13),          # every ref pixel >= 0.5: min(ref * 2 - 1) >= 0, PSNR's data_range 1
    "identical": (2, 64, "identical", 14),    # SSIM 1, PSNR inf, LPIPS 0
    "constant": (2, 64, "constant", 15),      # flat frames: every window has zero variance
    "batch33": (33, 64, "noisy", 16),         # PerceptualMetric.calculate_score: chunks of 32 and 1
}
ALEX_SHAPES = ((64, 3, 11), (192, 64, 5), (384, 192, 3), (256, 384, 3), (256, 256, 3))
LIN_CH = (64, 192, 384, 256, 256)


def _smooth(rng, n, size):
    low = rng.random((n, 3, size // 8, size // 8), dtype=np.float32)
    up = np.repeat(np.repeat(low, 8, axis=2), 8, axis=3).astype(np.float64)
    return uniform_filter(up, size=(1, 1, 9, 9)).astype(np.float32)


def make_case(name):
    """-> (preds, gts) float32 [n,3,s,s] in [0,1]."""
    n, s, kind, seed = CASES[name]
    rng = np.random.default_rng(seed)
    if kind == "constant":
        gts = np.broadcast_to(rng.random((n, 3, 1, 1), dtype=np.float32), (n, 3, s, s)).copy()
        preds = np.broadcast_to(rng.random((n, 3, 1, 1), dtype=np.float32), (n, 3, s, s)).copy()
        return preds, gts
    gts = _smooth(rng, n, s)
    if kind == "nonneg":
        gts = (np.float32(0.5) + np.float32(0.5) * gts).astype(np.float32)
    noise = (rng.random(gts.shape, dtype=np.float32) - np.float32(0.5)) * np.float32(0.2)
    preds = np.clip(gts + noise, 0, 1).astype(np.float32)
    if kind == "identical":
        preds = gts.copy()
    return preds, gts


def synthetic_alexnet(seed=5):
    """[(w, b)] float32 of the 5 AlexNet feature convolutions: uniform with He-uniform bounds, biases in +-0.05."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for cout, cin, k in ALEX_SHAPES:
        bound = float(np.sqrt(6.0 / (cin * k * k)))
        w = (torch.rand((cout, cin, k, k), generator=g) * 2 - 1) * bound
        b = (torch.rand(cout, generator=g) * 2 - 1) * 0.05
        out.append((w, b))
    return out


def synthetic_lins(seed=6):
    """lin0..lin4 weights [c] >= 0 (the published ones are non-negative)."""
    g = torch.Generator().manual_seed(seed)
    return [torch.rand(c, generator=g) * 0.2 for c in LIN_CH]


def alexnet_state_dict(convs):
    """torchvision alexnet().features keys."""
    sd = {}
    for (w, b), idx in zip(convs, (0, 3, 6, 8, 10)):
        sd["features.%d.weight" % idx], sd["features.%d.bias" % idx] = w, b
    return sd


def lin_state_dict(lins):
    return {"lin%d.model.1.weight" % k: l.view(1, -1, 1, 1) for k, l in enumerate(lins)}


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a.numpy() if torch.is_tensor(a) else a).tobytes())
    return h.hexdigest()
