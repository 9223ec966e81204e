"""Seeded inputs of the IS / FID tests (tests/golden/make_inception_golden.py, test_inception_cpu.py, test_inception_gpu.py).

Frames, synthetic InceptionV3 conv weights, BatchNorm affines and the Frechet feature sets are regenerated from their
seeds with uniform draws, box filters, clipping and elementwise arithmetic only (no BLAS, no transcendental functions,
so every host makes the same bytes); the golden pins them by SHA-256.  The BatchNorm running statistics are not
regenerated: they were calibrated once on a seeded batch (so activations stay O(1) through all 94 layers) and live in
tests/golden/inception.npz.  Frames are [N,3,H,W] float32 in [0,1], the metric classes' input.
"""
import hashlib

import numpy as np
import torch
from scipy.ndimage import uniform_filter

from impersonator_b200.metrics import INCEPTION_CONVS

# name -> (n, h, w, seed)
CASES = {
    "rand256": (2, 256, 256, 21),
    "rand512": (1, 512, 512, 22),
    "ident299": (1, 299, 299, 23),            # the resize is the identity
    "wide": (1, 184, 328, 24),                # non-square, upsampled rows and columns by different factors
}
CALIB = (4, 299, 299, 20)                     # the batch the BatchNorm statistics were calibrated on
BATCH33 = (33, 64, 64, 25)                    # calculate_score: chunks of 32 and 1 (preds, then gts with seed + 100)
# Frechet feature sets: name -> (n, d, seed); the reference's fid_score_func of (pred, gt) and is_score_func of the
# softmax of IS_GAIN * pred are in the golden
FEATS = {
    "d2048_n4096": (4096, 2048, 31),
    "d2048_n200": (200, 2048, 32),            # n < d: rank-deficient covariances
    "d64_n500": (500, 64, 33),
    "d8_n50": (50, 8, 34),
}
IS_GAIN = 4.0


def make_frames(n, h, w, seed):
    """Smooth random frames plus noise, float32 [n,3,h,w] in [0,1]."""
    rng = np.random.default_rng(seed)
    low = rng.random((n, 3, -(-h // 8), -(-w // 8)), dtype=np.float32)
    up = np.repeat(np.repeat(low, 8, axis=2), 8, axis=3)[:, :, :h, :w].astype(np.float64)
    img = uniform_filter(up, size=(1, 1, 9, 9)).astype(np.float32)
    noise = (rng.random(img.shape, dtype=np.float32) - np.float32(0.5)) * np.float32(0.2)
    return np.clip(img + noise, 0, 1).astype(np.float32)


def make_case(name):
    return make_frames(*CASES[name])


def make_batch33():
    n, h, w, seed = BATCH33
    return make_frames(n, h, w, seed), make_frames(n, h, w, seed + 100)


def synthetic_inception(seed=7):
    """{name: (w, gamma, beta)} float32 of the 94 BasicConv2d: He-uniform conv weights, gamma in [0.2, 0.5), beta in
    [0.5, 1.0).  With the calibrated statistics most pre-activations are positive, so the network is close to linear
    and a 1e-5 change of the input moves the features by about 1e-5 of their maximum; gamma in [0.5, 1.5) with beta
    around 0 makes a chaotic network that amplifies the same change 160-fold."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, (cin, cout, kh, kw, _, _, _) in INCEPTION_CONVS.items():
        bound = float(np.sqrt(6.0 / (cin * kh * kw)))
        w = (torch.rand((cout, cin, kh, kw), generator=g) * 2 - 1) * bound
        gamma = torch.rand(cout, generator=g) * 0.3 + 0.2
        beta = torch.rand(cout, generator=g) * 0.5 + 0.5
        out[name] = (w, gamma, beta)
    return out


def state_dict(params, stats):
    """torchvision Inception3 keys of the used modules.  stats: {name + '/mean' | '/var': float32 [cout]} (the golden's
    calibrated running statistics)."""
    sd = {}
    for name, (w, gamma, beta) in params.items():
        sd[name + ".conv.weight"] = w
        sd[name + ".bn.weight"], sd[name + ".bn.bias"] = gamma, beta
        sd[name + ".bn.running_mean"] = torch.as_tensor(np.asarray(stats[name + "/mean"]))
        sd[name + ".bn.running_var"] = torch.as_tensor(np.asarray(stats[name + "/var"]))
    return sd


def golden_state_dict(gold):
    return state_dict(synthetic_inception(), {k[3:]: gold[k] for k in gold.files if k.startswith("bn/")})


def make_feats(name):
    """-> (pred, gt) float64 [n,d]: per-dimension scales and offsets plus a shared 16-factor component (elementwise,
    so the covariances are not diagonal)."""
    n, d, seed = FEATS[name]
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(2):
        scale = 0.5 + rng.random(d)
        shift = rng.random(d) * 2
        mix = rng.random(d) - 0.5
        z = rng.random((n, 16))
        x = rng.random((n, d)) * scale + shift
        x += z[:, np.arange(d) % 16] * mix
        out.append(x)
    return out[0], out[1]


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a.numpy() if torch.is_tensor(a) else a).tobytes())
    return h.hexdigest()
