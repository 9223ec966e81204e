"""Paired image-quality metrics of his_evaluators (metrics/metrics.py:450-631) on this library's kernels.

``SSIMMetric``, ``PSNRMetric`` and ``PerceptualMetric`` have the reference's constructors, ``forward``,
``calculate_score`` and ``quality``, and take the same inputs: [N,3,H,W] (or one [3,H,W]) float32 frames in [0,1], numpy
or torch.  CUDA tensors are scored where they are; anything else is copied to the device once.

  SSIM / PSNR   skimage 0.16.2 structural_similarity(multichannel=True) / peak_signal_noise_ratio of the [-1,1] HWC
                images, both in one lwb_ssim_psnr call per batch (fp64 per-frame scores)
  LPIPS         v0.1 net-lin AlexNet (lpips/models/networks_basic.py:65-168, pretrained_networks.py:58-96):
                  scaling layer of pred and ref as one batch of 2N          lwb_lpips_input
                  conv1 11x11 s4 p2 + ReLU                                  lwb_conv2d_direct_relu_nhwc (fp32)
                  max_pool(3, 2)                                            lwb_maxpool_nhwc (floor mode)
                  conv2 5x5 / conv3..5 3x3 + bias + ReLU                    the conv engine in fp16x3 + lwb_det_bias_act
                  per tap: normalise, squared difference, lin, mean         lwb_lpips_layer

Weights: AlexNet from torchvision's ``alexnet-owt-7be5be79.pth`` in ``<torch.hub.get_dir()>/checkpoints/`` (or
``weights=``, a path or state dict); the ``lin`` layers from his_evaluators' ``lpips/weights/v0.1/alex.pth`` (or
``lin_weights=``).  Nothing is ever downloaded.
"""
import importlib.util
import math
import os

import numpy as np
import torch

from . import kernels as K
from ._lib import LwbError

ALEXNET_FILE = "alexnet-owt-7be5be79.pth"
LIN_FILE = os.path.join("lpips", "weights", "v0.1", "alex.pth")
SPLIT = 1                                                            # fp16x3, as the detector
# (features index, cin, cout, k, stride, pad) of torchvision's alexnet().features up to relu5
ALEX_CONVS = ((0, 3, 64, 11, 4, 2), (3, 64, 192, 5, 1, 2), (6, 192, 384, 3, 1, 1), (8, 384, 256, 3, 1, 1),
              (10, 256, 256, 3, 1, 1))
HIGHER = 'higher score is better'                                    # metrics.py:179-180
LOWER = 'lower score is better.'


def _frames(x, device):
    """[N,3,H,W] or [3,H,W] numpy / tensor -> contiguous float32 CUDA tensor [N,3,H,W] (no copy for one already there)."""
    t = torch.as_tensor(x)
    if t.dim() == 3:
        t = t[None]
    if t.dim() != 4 or t.shape[1] != 3:
        raise LwbError("frames must be [N,3,H,W] or [3,H,W], got %s" % (tuple(t.shape),))
    if not t.is_cuda:
        t = t.to(device)
    return t.float().contiguous()


def _device(device):
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    if dev.type != "cuda":
        raise LwbError("the metrics run on CUDA devices only (no CPU path), got %s" % dev)
    return dev


def ssim_psnr(pred, ref, from01=True):
    """Per-frame (SSIM, PSNR) fp64 CUDA tensors [N] of two frame batches."""
    dev = pred.device if torch.is_tensor(pred) and pred.is_cuda else _device(None)
    p, r = _frames(pred, dev), _frames(ref, dev)
    with torch.cuda.device(dev):
        return K.ssim_psnr(p, r, from01=from01)


class SSIMMetric(object):
    def __init__(self, device=None):
        self.device = device

    def forward(self, pred, ref):
        """One frame [3,H,W] in [0,1] -> float."""
        return float(ssim_psnr(pred, ref)[0][0].item())

    def calculate_score(self, preds, gts):
        assert len(preds) == len(gts)
        return float(np.mean(ssim_psnr(preds, gts)[0].cpu().numpy()))

    def quality(self):
        return HIGHER


class PSNRMetric(object):
    def __init__(self, device=None):
        self.device = device

    def forward(self, pred, ref):
        return float(ssim_psnr(pred, ref)[1][0].item())

    def calculate_score(self, preds, gts):
        assert len(preds) == len(gts)
        return float(np.mean(ssim_psnr(preds, gts)[1].cpu().numpy()))

    def quality(self):
        return HIGHER


# ---- LPIPS -----------------------------------------------------------------------------------------------------------
def default_alexnet_path():
    return os.path.join(torch.hub.get_dir(), "checkpoints", ALEXNET_FILE)


def default_lin_path():
    """his_evaluators' lpips/weights/v0.1/alex.pth, when that package is installed (found without importing it)."""
    spec = importlib.util.find_spec("his_evaluators")
    if spec is None or not spec.submodule_search_locations:
        return None
    return os.path.join(list(spec.submodule_search_locations)[0], "metrics", LIN_FILE)


def _load(weights, default, what):
    if isinstance(weights, dict):
        return weights
    path = weights if weights is not None else default
    if path is None or not os.path.exists(path):
        raise LwbError("%s not found%s: pass its path or state dict (this package never downloads)"
                       % (what, " at %s" % path if path else ""))
    return torch.load(path, map_location="cpu", weights_only=True)


def load_alexnet_weights(weights=None):
    """-> [(w, b)] of the 5 convolutions of torchvision's alexnet().features (state dict, path or the hub cache)."""
    sd = _load(weights, default_alexnet_path(), "torchvision AlexNet weights (%s)" % ALEXNET_FILE)
    out = []
    for idx, cin, cout, k, _, _ in ALEX_CONVS:
        w, b = sd.get("features.%d.weight" % idx), sd.get("features.%d.bias" % idx)
        if w is None or b is None or tuple(w.shape) != (cout, cin, k, k):
            raise LwbError("AlexNet state dict: features.%d must be a %dx%d conv %d -> %d with bias" % (idx, k, k, cin, cout))
        out.append((w.float(), b.float()))
    return out


def load_lin_weights(lin_weights=None):
    """-> [lin_k [c_k]] of PNetLin's lin0..lin4 (``lin{k}.model.1.weight`` [1,c,1,1])."""
    sd = _load(lin_weights, default_lin_path(), "LPIPS lin weights (his_evaluators %s)" % LIN_FILE)
    out = []
    for k, (_, _, c, _, _, _) in enumerate(ALEX_CONVS):
        w = sd.get("lin%d.model.1.weight" % k)
        if w is None or w.numel() != c:
            raise LwbError("LPIPS lin state dict: lin%d.model.1.weight must hold %d weights" % (k, c))
        out.append(w.float().reshape(c))
    return out


class _AlexStream(object):
    """AlexNet features + LPIPS taps bound to (N pairs, H, W): buffers, conv plans and weights on the device."""

    def __init__(self, convs, lins, n, h, w, dev):
        self.n, self.h, self.w = n, h, w
        n2 = 2 * n
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        ops = lambda *s: (torch.empty(s, dtype=torch.float16, device=dev), torch.empty(s, dtype=torch.float16, device=dev))
        self.x = f(n2, 3, h, w)
        self.w1 = convs[0][0].to(dev).contiguous()
        self.b1 = convs[0][1].to(dev).contiguous()
        h1, w1 = (h + 4 - 11) // 4 + 1, (w + 4 - 11) // 4 + 1
        hp1, wp1 = (h1 - 3) // 2 + 1, (w1 - 3) // 2 + 1
        hp2, wp2 = (hp1 - 3) // 2 + 1, (wp1 - 3) // 2 + 1
        if min(h1, w1) < 3 or min(hp1, wp1) < 3 or min(hp2, wp2) < 1:
            raise LwbError("LPIPS: %dx%d frames are too small for AlexNet's features" % (h, w))
        self.feats = [f(n2, h1, w1, 64), f(n2, hp1, wp1, 192), f(n2, hp2, wp2, 384), f(n2, hp2, wp2, 256), f(n2, hp2, wp2, 256)]
        self.pool1, self.pool2 = ops(n2, hp1, wp1, 64), ops(n2, hp2, wp2, 192)
        self.a3, self.a4 = ops(n2, hp2, wp2, 384), ops(n2, hp2, wp2, 256)
        ins = (self.pool1, self.pool2, self.a3, self.a4)
        outs = (None, None, self.a3, self.a4, None)
        amax = torch.stack([c[0].abs().max() for c in convs[1:]]).tolist()
        self.layers = []
        for k in range(1, 5):
            _, cin, cout, ks, _, pad = ALEX_CONVS[k]
            x_pair = ins[k - 1]
            hh, ww = x_pair[0].shape[1:3]
            d = K.make_conv_desc(n2, hh, ww, cin, cout, ks, ks, pad=pad, split=SPLIT)
            raw = f(n2, d.h_out, d.w_out, cout)
            wp = K.pack_conv_weight(convs[k][0].to(dev), split=SPLIT, absmax=amax[k - 1])
            plan = K.ConvPlan(d, x_pair, None, wp, raw, None)
            self.layers.append(dict(plan=plan, raw=raw, bias=convs[k][1].to(dev).contiguous(), out=outs[k]))
        self.lins = [l.to(dev).contiguous() for l in lins]
        self.layer_vals = torch.empty((n, 5), dtype=torch.float32, device=dev)
        self.score = torch.empty(n, dtype=torch.float32, device=dev)

    def run(self, pred, ref, from01):
        """-> (score [N], per-layer values [N,5]) device views, valid until the next run."""
        K.lpips_input(pred, ref, from01=from01, out=self.x)
        K.conv2d_direct_relu_nhwc(self.x, self.w1, self.b1, stride=4, pad=2, out=self.feats[0])
        K.maxpool_nhwc(self.feats[0], 3, 2, y_hi=self.pool1[0], y_lo=self.pool1[1])
        for k, L in enumerate(self.layers):
            L["plan"].run()
            o = L["out"]
            K.det_bias_act(L["raw"], L["bias"], relu=True, y_f32=self.feats[k + 1], y_hi=o[0] if o else None,
                           y_lo=o[1] if o else None)
            if k == 0:
                K.maxpool_nhwc(self.feats[1], 3, 2, y_hi=self.pool2[0], y_lo=self.pool2[1])
        for k in range(5):
            K.lpips_layer(self.feats[k], self.lins[k], k, self.layer_vals, self.score)
        return self.score, self.layer_vals


class LPIPS(object):
    """PNetLin(pnet_type='alex', version='0.1') of his_evaluators on the device."""

    def __init__(self, device=None, weights=None, lin_weights=None):
        self.device = _device(device)
        self.convs = load_alexnet_weights(weights)
        self.lins = load_lin_weights(lin_weights)
        self._streams = {}

    def __call__(self, pred, ref, from01=True):
        """-> (per-frame score [N] fp32, per-layer values [N,5]) device tensors (fresh copies)."""
        p, r = _frames(pred, self.device), _frames(ref, self.device)
        if p.shape != r.shape:
            raise LwbError("pred %s and ref %s differ in shape" % (tuple(p.shape), tuple(r.shape)))
        n, _, h, w = p.shape
        key = (n, h, w)
        with torch.cuda.device(self.device):
            st = self._streams.get(key)
            if st is None:
                while len(self._streams) >= 2:
                    self._streams.pop(next(iter(self._streams)))
                st = self._streams[key] = _AlexStream(self.convs, self.lins, n, h, w, self.device)
            score, layers = st.run(p, r, from01)
            return score.clone(), layers.clone()


class PerceptualMetric(object):
    """metrics.py:569-631 (LPIPS, lower is better)."""

    def __init__(self, device=None, weights=None, lin_weights=None):
        self.device = _device(device)
        self.lpips = LPIPS(self.device, weights, lin_weights)

    def forward(self, pred, ref):
        """Mean LPIPS of a batch (a 0-d float32 CUDA tensor, as the reference's torch.mean)."""
        return self.lpips(pred, ref)[0].mean()

    def calculate_score(self, preds, gts, batch_size=32):
        """The mean of the per-``batch_size``-chunk means (a shorter last chunk weighs more, as in the reference)."""
        assert len(preds) == len(gts)
        length = len(preds)
        scores = []
        for i in range(int(math.ceil(length / batch_size))):
            s = self.lpips(preds[i * batch_size: (i + 1) * batch_size], gts[i * batch_size: (i + 1) * batch_size])[0]
            scores.append(s.mean())
        return torch.mean(torch.stack(scores)).cpu().numpy()

    def quality(self):
        return LOWER


def score_frames(pred, ref, from01=False, lpips=None):
    """Per-frame scores of two [N,3,H,W] CUDA frame batches (in [-1,1] unless from01) without leaving the device:
    dict(ssim fp64 [N], psnr fp64 [N], lpips fp32 [N] when an ``LPIPS`` is given)."""
    s, p = K.ssim_psnr(_frames(pred, pred.device), _frames(ref, pred.device), from01=from01)
    out = dict(ssim=s, psnr=p)
    if lpips is not None:
        out["lpips"] = lpips(pred, ref, from01=from01)[0]
    return out
