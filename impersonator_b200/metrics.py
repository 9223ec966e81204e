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

The unpaired metrics ``InceptionScoreMetric`` and ``FIDMetric`` (metrics.py:634-781) share one ``InceptionFeatures``
per device: torchvision's InceptionV3 up to its 2048 pool features (lwb_inception_input, the direct stem, the conv
engine in fp16x3 with lwb_bn_act_segment, the NHWC max / average pools); the scores are float64 torch on the device.
"""
import functools
import importlib.util
import math
import os

import numpy as np
import torch

from . import kernels as K
from ._lib import LwbError
from .binding import Conv, Operands, PlanBinder, bn_affine, stream_for

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

    def __init__(self, owner, n, h, w, dev):
        self.n, self.h, self.w = n, h, w
        convs, lins = owner.convs, owner.lins
        n2 = 2 * n
        f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        self.x = f(n2, 3, h, w)
        self.w1 = convs[0][0].to(dev).contiguous()
        self.b1 = convs[0][1].to(dev).contiguous()
        h1, w1 = (h + 4 - 11) // 4 + 1, (w + 4 - 11) // 4 + 1
        hp1, wp1 = (h1 - 3) // 2 + 1, (w1 - 3) // 2 + 1
        hp2, wp2 = (hp1 - 3) // 2 + 1, (wp1 - 3) // 2 + 1
        if min(h1, w1) < 3 or min(hp1, wp1) < 3 or min(hp2, wp2) < 1:
            raise LwbError("LPIPS: %dx%d frames are too small for AlexNet's features" % (h, w))
        self.feats = [f(n2, h1, w1, 64), f(n2, hp1, wp1, 192), f(n2, hp2, wp2, 384), f(n2, hp2, wp2, 256), f(n2, hp2, wp2, 256)]
        self.pool1, self.pool2 = Operands((n2, hp1, wp1, 64), dev, SPLIT), Operands((n2, hp2, wp2, 192), dev, SPLIT)
        self.a3, self.a4 = Operands((n2, hp2, wp2, 384), dev, SPLIT), Operands((n2, hp2, wp2, 256), dev, SPLIT)
        ins = (self.pool1, self.pool2, self.a3, self.a4)
        outs = (None, None, self.a3, self.a4, None)
        plans = PlanBinder(dev, SPLIT)
        self.layers = []
        for k in range(1, 5):
            pad = ALEX_CONVS[k][5]
            hh, ww = ins[k - 1].hi.shape[1:3]
            conv = plans.conv(convs[k][0].to(dev), ins[k - 1].pair, n2, hh, ww, pad=pad)
            self.layers.append(dict(conv=conv, bias=convs[k][1].to(dev).contiguous(), out=outs[k]))
        plans.finalize()
        self.lins = [l.to(dev).contiguous() for l in lins]
        self.layer_vals = torch.empty((n, 5), dtype=torch.float32, device=dev)
        self.score = torch.empty(n, dtype=torch.float32, device=dev)

    def run(self, pred, ref, from01):
        """-> (score [N], per-layer values [N,5]) device views, valid until the next run."""
        K.lpips_input(pred, ref, from01=from01, out=self.x)
        K.conv2d_direct_relu_nhwc(self.x, self.w1, self.b1, stride=4, pad=2, out=self.feats[0])
        K.maxpool_nhwc(self.feats[0], 3, 2, y_hi=self.pool1.hi, y_lo=self.pool1.lo)
        for k, L in enumerate(self.layers):
            L["conv"].plan.run()
            o = L["out"]
            K.det_bias_act(L["conv"].out, L["bias"], relu=True, y_f32=self.feats[k + 1], y_hi=o.hi if o else None,
                           y_lo=o.lo if o else None)
            if k == 0:
                K.maxpool_nhwc(self.feats[1], 3, 2, y_hi=self.pool2.hi, y_lo=self.pool2.lo)
        for k in range(5):
            K.lpips_layer(self.feats[k], self.lins[k], k, self.layer_vals, self.score)
        return self.score, self.layer_vals


class LPIPS(object):
    """PNetLin(pnet_type='alex', version='0.1') of his_evaluators on the device."""

    def __init__(self, device=None, weights=None, lin_weights=None):
        self.device = _device(device)
        self.convs = load_alexnet_weights(weights)
        self.lins = load_lin_weights(lin_weights)

    def __call__(self, pred, ref, from01=True):
        """-> (per-frame score [N] fp32, per-layer values [N,5]) device tensors (fresh copies)."""
        p, r = _frames(pred, self.device), _frames(ref, self.device)
        if p.shape != r.shape:
            raise LwbError("pred %s and ref %s differ in shape" % (tuple(p.shape), tuple(r.shape)))
        n, _, h, w = p.shape
        with torch.cuda.device(self.device):
            st = stream_for(self, _AlexStream, (n, h, w), n, h, w, self.device, limit=2)
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


# ---- IS / FID: InceptionV3 features ----------------------------------------------------------------------------------
# torchvision's current Inception3 checkpoint, then the one torchvision 0.4.0 (his_evaluators' pin) caches
INCEPTION_FILES = ("inception_v3_google-0cc3c7bd.pth", "inception_v3_google-1a9a5a14.pth")
BN_EPS = 0.001                                                      # torchvision BasicConv2d


def _inception_convs():
    """name -> (cin, cout, kh, kw, stride, pad_h, pad_w) of the 94 BasicConv2d of torchvision's Inception3 up to
    Mixed_7c (the modules InceptionV3(output_blocks=[3]) runs; AuxLogits and fc are never used)."""
    L = {}

    def c(name, cin, cout, k, s=1, p=0):
        kh, kw = k if isinstance(k, tuple) else (k, k)
        ph, pw = p if isinstance(p, tuple) else (p, p)
        L[name] = (cin, cout, kh, kw, s, ph, pw)

    c("Conv2d_1a_3x3", 3, 32, 3, 2)
    c("Conv2d_2a_3x3", 32, 32, 3)
    c("Conv2d_2b_3x3", 32, 64, 3, p=1)
    c("Conv2d_3b_1x1", 64, 80, 1)
    c("Conv2d_4a_3x3", 80, 192, 3)
    for b, cin, pf in (("Mixed_5b", 192, 32), ("Mixed_5c", 256, 64), ("Mixed_5d", 288, 64)):
        c(b + ".branch1x1", cin, 64, 1)
        c(b + ".branch5x5_1", cin, 48, 1)
        c(b + ".branch5x5_2", 48, 64, 5, p=2)
        c(b + ".branch3x3dbl_1", cin, 64, 1)
        c(b + ".branch3x3dbl_2", 64, 96, 3, p=1)
        c(b + ".branch3x3dbl_3", 96, 96, 3, p=1)
        c(b + ".branch_pool", cin, pf, 1)
    c("Mixed_6a.branch3x3", 288, 384, 3, 2)
    c("Mixed_6a.branch3x3dbl_1", 288, 64, 1)
    c("Mixed_6a.branch3x3dbl_2", 64, 96, 3, p=1)
    c("Mixed_6a.branch3x3dbl_3", 96, 96, 3, 2)
    for b, c7 in (("Mixed_6b", 128), ("Mixed_6c", 160), ("Mixed_6d", 160), ("Mixed_6e", 192)):
        c(b + ".branch1x1", 768, 192, 1)
        c(b + ".branch7x7_1", 768, c7, 1)
        c(b + ".branch7x7_2", c7, c7, (1, 7), p=(0, 3))
        c(b + ".branch7x7_3", c7, 192, (7, 1), p=(3, 0))
        c(b + ".branch7x7dbl_1", 768, c7, 1)
        c(b + ".branch7x7dbl_2", c7, c7, (7, 1), p=(3, 0))
        c(b + ".branch7x7dbl_3", c7, c7, (1, 7), p=(0, 3))
        c(b + ".branch7x7dbl_4", c7, c7, (7, 1), p=(3, 0))
        c(b + ".branch7x7dbl_5", c7, 192, (1, 7), p=(0, 3))
        c(b + ".branch_pool", 768, 192, 1)
    c("Mixed_7a.branch3x3_1", 768, 192, 1)
    c("Mixed_7a.branch3x3_2", 192, 320, 3, 2)
    c("Mixed_7a.branch7x7x3_1", 768, 192, 1)
    c("Mixed_7a.branch7x7x3_2", 192, 192, (1, 7), p=(0, 3))
    c("Mixed_7a.branch7x7x3_3", 192, 192, (7, 1), p=(3, 0))
    c("Mixed_7a.branch7x7x3_4", 192, 192, 3, 2)
    for b, cin in (("Mixed_7b", 1280), ("Mixed_7c", 2048)):
        c(b + ".branch1x1", cin, 320, 1)
        c(b + ".branch3x3_1", cin, 384, 1)
        c(b + ".branch3x3_2a", 384, 384, (1, 3), p=(0, 1))
        c(b + ".branch3x3_2b", 384, 384, (3, 1), p=(1, 0))
        c(b + ".branch3x3dbl_1", cin, 448, 1)
        c(b + ".branch3x3dbl_2", 448, 384, 3, p=1)
        c(b + ".branch3x3dbl_3a", 384, 384, (1, 3), p=(0, 1))
        c(b + ".branch3x3dbl_3b", 384, 384, (3, 1), p=(1, 0))
        c(b + ".branch_pool", cin, 192, 1)
    return L


INCEPTION_CONVS = _inception_convs()


def default_inception_paths():
    ck = os.path.join(torch.hub.get_dir(), "checkpoints")
    return [os.path.join(ck, f) for f in INCEPTION_FILES]


def load_inception_weights(weights=None):
    """-> {name: (w [cout,cin,kh,kw] fp32, bn scale [cout], bn shift [cout])} of the 94 BasicConv2d: the eval-mode
    BatchNorm as the per-channel affine scale = gamma / sqrt(var + 0.001), shift = beta - mean * scale (in float64,
    stored fp32).  ``weights``: a torchvision Inception3 state dict or its path; by default the first of
    INCEPTION_FILES found in ``<torch.hub.get_dir()>/checkpoints/``."""
    if weights is None:
        found = [p for p in default_inception_paths() if os.path.exists(p)]
        if not found:
            raise LwbError("torchvision InceptionV3 weights not found (looked for %s): pass their path or state dict "
                           "(this package never downloads)" % " and ".join(default_inception_paths()))
        weights = found[0]
    sd = _load(weights, None, "torchvision InceptionV3 weights (%s)" % INCEPTION_FILES[0])
    out = {}
    for name, (cin, cout, kh, kw, _, _, _) in INCEPTION_CONVS.items():
        w = sd.get(name + ".conv.weight")
        if w is None or tuple(w.shape) != (cout, cin, kh, kw):
            raise LwbError("InceptionV3 state dict: %s.conv.weight must be [%d,%d,%d,%d], got %s"
                           % (name, cout, cin, kh, kw, None if w is None else tuple(w.shape)))
        bn = []
        for k in ("weight", "bias", "running_mean", "running_var"):
            t = sd.get("%s.bn.%s" % (name, k))
            if t is None or tuple(t.shape) != (cout,):
                raise LwbError("InceptionV3 state dict: %s.bn.%s must hold %d values" % (name, k, cout))
            bn.append(t)
        out[name] = (w.float(),) + bn_affine(*bn, BN_EPS)
    return out


def _up64(c):
    return (c + 63) // 64 * 64


class _InceptionStream(object):
    """InceptionV3(output_blocks=[3]) features bound to (N, H, W): buffers, conv plans and the launch list.

    Every convolution but the stem runs on the conv engine in fp16x3 with its input channels zero padded to a multiple
    of 64; the same-input 1x1 convolutions of each Mixed block (pool branch included) are one GEMM whose columns
    lwb_bn_act_segment splits into the branches.  The fp32 copies of Conv2d_2b/4a and of Mixed_5d/6e feed the max
    pools; stem / mixed_5d / mixed_6e are kept for inspection."""

    def __init__(self, net, n, h, w, dev):
        self.n, self.dev, self.net = n, dev, net
        self.ops = []
        self._plans = PlanBinder(dev, SPLIT)
        self.x = self._f32(n, 3, 299, 299)
        # Conv2d_1a (BN folded into the fp32 stem) -> operands of 64 channels
        self.stem = self._f32(n, 149, 149, 32)
        self.ops.append(lambda: K.conv2d_direct_relu_nhwc(self.x, net.stem_w, net.stem_b, stride=2, out=self.stem))
        a = Operands((n, 149, 149, 64), self.dev, SPLIT)
        self._seg(self.stem, 0, None, a, 0, relu=False, c=32, c_out=64)
        a = self._single("Conv2d_2a_3x3", a)
        b2 = self._f32(n, 147, 147, 64)
        self._single("Conv2d_2b_3x3", a, f32=b2)
        a = Operands((n, 73, 73, 64), self.dev, SPLIT)
        self.ops.append(functools.partial(K.maxpool_nhwc, b2, 3, 2, y_hi=a.hi, y_lo=a.lo))
        a = self._single("Conv2d_3b_1x1", a)
        b4 = self._f32(n, 71, 71, 192)
        self._single("Conv2d_4a_3x3", a, f32=b4)
        a = Operands((n, 35, 35, 192), self.dev, SPLIT)
        self.ops.append(functools.partial(K.maxpool_nhwc, b4, 3, 2, y_hi=a.hi, y_lo=a.lo))
        a = self._block_a("Mixed_5b", a)
        a = self._block_a("Mixed_5c", a)
        self.mixed_5d = self._f32(n, 35, 35, 320)
        a = self._block_a("Mixed_5d", a, f32=self.mixed_5d)
        a = self._block_b("Mixed_6a", a, self.mixed_5d, 288)
        for b in ("Mixed_6b", "Mixed_6c", "Mixed_6d"):
            a = self._block_c(b, a)
        self.mixed_6e = self._f32(n, 17, 17, 768)
        a = self._block_c("Mixed_6e", a, f32=self.mixed_6e)
        a = self._block_d("Mixed_7a", a, self.mixed_6e)
        a = self._block_e("Mixed_7b", a)
        self.feats = self._f32(n, 2048)
        self._block_e("Mixed_7c", a, feats=self.feats)
        self._plans.finalize()
        del self._plans
        self.ops = [op.plan.run if isinstance(op, Conv) else op for op in self.ops]

    # -- buffers and launches --
    def _f32(self, *s):
        return torch.empty(s, dtype=torch.float32, device=self.dev)

    def _conv(self, names, x):
        """One conv-engine GEMM of the same-input, same-shape convolutions ``names`` over operands x [n,h,w,64k]
        -> (raw fp32 [n,ho,wo,up64(sum cout)], {name: first column})."""
        specs = [INCEPTION_CONVS[nm] for nm in names]
        _, _, kh, kw, s, ph, pw = specs[0]
        if any(sp[2:] != specs[0][2:] for sp in specs):
            raise LwbError("merged convolutions must share kernel, stride and padding: %s" % (names,))
        n, h, w, cp = x.hi.shape
        cols, c0 = {}, 0
        for nm, sp in zip(names, specs):
            cols[nm] = c0
            c0 += sp[1]
        wt = torch.cat([self.net.convs[nm][0] for nm in names], 0).to(self.dev)
        conv = self._plans.conv(wt, x.pair, n, h, w, stride=s, pad=ph, pad_w=pw, cout_pad=_up64(c0), cin_pad=cp)
        self.ops.append(conv)                            # its plan.run once finalize() has made the plan
        return conv.out, cols

    def _seg(self, raw, c0, name, y, off, relu=True, c=None, c_out=None, box=False, f32=None):
        """Branch ``name`` (columns c0.. of raw) -> BN + ReLU into channels off.. of operands y and / or fp32 f32."""
        scale = shift = None
        if name is not None:
            _, scale, shift = self.net.convs[name]
            scale, shift = scale.to(self.dev), shift.to(self.dev)
            c = INCEPTION_CONVS[name][1]
        hi, lo = y.pair if y is not None else (None, None)
        self.ops.append(lambda: K.bn_act_segment(raw, c0, c, scale, shift, relu=relu, box=box, c_out=c_out, y_f32=f32,
                                                 y_hi=hi, y_lo=lo, off_y=off))

    def _single(self, name, x, f32=None, y=None, off=0):
        """One convolution + BN + ReLU into channels off.. of y / f32, or into new operands of up64(cout) channels
        (the pad channels zeroed) when neither is given."""
        raw, _ = self._conv([name], x)
        cout = INCEPTION_CONVS[name][1]
        c_out = cout
        if y is None and f32 is None:
            c_out = _up64(cout)
            y = Operands((*raw.shape[:3], c_out), self.dev, SPLIT)
        self._seg(raw, 0, name, y, off, c_out=c_out, f32=f32)
        return y

    def _gap(self, raw, name, off):
        """Mixed_7c branch -> BN + ReLU + the spatial mean straight into feats[:, off:]."""
        _, scale, shift = self.net.convs[name]
        scale, shift = scale.to(self.dev), shift.to(self.dev)
        self.ops.append(lambda: K.global_avgpool_nhwc(raw, scale, shift, relu=True, out=self.feats[:, off:], ld_out=2048))

    # -- the Inception blocks (torchvision inception.py InceptionA..E) --
    def _block_a(self, b, x, f32=None):
        n, h, w, _ = x.hi.shape
        raw, col = self._conv([b + ".branch1x1", b + ".branch5x5_1", b + ".branch3x3dbl_1", b + ".branch_pool"], x)
        pf = INCEPTION_CONVS[b + ".branch_pool"][1]
        pitch = _up64(224 + pf)
        out = Operands((n, h, w, pitch), self.dev, SPLIT)
        t5, td = Operands((n, h, w, 64), self.dev, SPLIT), Operands((n, h, w, 64), self.dev, SPLIT)
        self._seg(raw, col[b + ".branch1x1"], b + ".branch1x1", out, 0, f32=f32)
        self._seg(raw, col[b + ".branch5x5_1"], b + ".branch5x5_1", t5, 0, c_out=64)
        self._seg(raw, col[b + ".branch3x3dbl_1"], b + ".branch3x3dbl_1", td, 0)
        self._seg(raw, col[b + ".branch_pool"], b + ".branch_pool", out, 224, c_out=pitch - 224, box=True, f32=f32)
        self._single(b + ".branch5x5_2", t5, y=out, off=64, f32=f32)
        td = self._single(b + ".branch3x3dbl_2", td)
        self._single(b + ".branch3x3dbl_3", td, y=out, off=128, f32=f32)
        return out

    def _block_b(self, b, x, x_f32, cin):
        n = x.hi.shape[0]
        out = Operands((n, 17, 17, 768), self.dev, SPLIT)
        self._single(b + ".branch3x3", x, y=out, off=0)
        t = self._single(b + ".branch3x3dbl_1", x)
        t = self._single(b + ".branch3x3dbl_2", t)
        self._single(b + ".branch3x3dbl_3", t, y=out, off=384)
        self.ops.append(lambda: K.maxpool_nhwc_slice(x_f32, cin, 3, 2, y_hi=out.hi, y_lo=out.lo, off_y=480))
        return out

    def _block_c(self, b, x, f32=None):
        n, h, w, _ = x.hi.shape
        raw, col = self._conv([b + ".branch1x1", b + ".branch7x7_1", b + ".branch7x7dbl_1", b + ".branch_pool"], x)
        c7 = INCEPTION_CONVS[b + ".branch7x7_1"][1]
        out = Operands((n, h, w, 768), self.dev, SPLIT)
        ta, tb = Operands((n, h, w, _up64(c7)), self.dev, SPLIT), Operands((n, h, w, _up64(c7)), self.dev, SPLIT)
        self._seg(raw, col[b + ".branch1x1"], b + ".branch1x1", out, 0, f32=f32)
        self._seg(raw, col[b + ".branch7x7_1"], b + ".branch7x7_1", ta, 0, c_out=_up64(c7))
        self._seg(raw, col[b + ".branch7x7dbl_1"], b + ".branch7x7dbl_1", tb, 0, c_out=_up64(c7))
        self._seg(raw, col[b + ".branch_pool"], b + ".branch_pool", out, 576, box=True, f32=f32)
        ta = self._single(b + ".branch7x7_2", ta)
        self._single(b + ".branch7x7_3", ta, y=out, off=192, f32=f32)
        for k in (2, 3, 4):
            tb = self._single(b + ".branch7x7dbl_%d" % k, tb)
        self._single(b + ".branch7x7dbl_5", tb, y=out, off=384, f32=f32)
        return out

    def _block_d(self, b, x, x_f32):
        n = x.hi.shape[0]
        raw, col = self._conv([b + ".branch3x3_1", b + ".branch7x7x3_1"], x)
        out = Operands((n, 8, 8, 1280), self.dev, SPLIT)
        ta, tb = Operands((n, 17, 17, 192), self.dev, SPLIT), Operands((n, 17, 17, 192), self.dev, SPLIT)
        self._seg(raw, col[b + ".branch3x3_1"], b + ".branch3x3_1", ta, 0)
        self._seg(raw, col[b + ".branch7x7x3_1"], b + ".branch7x7x3_1", tb, 0)
        self._single(b + ".branch3x3_2", ta, y=out, off=0)
        tb = self._single(b + ".branch7x7x3_2", tb)
        tb = self._single(b + ".branch7x7x3_3", tb)
        self._single(b + ".branch7x7x3_4", tb, y=out, off=320)
        self.ops.append(lambda: K.maxpool_nhwc_slice(x_f32, 768, 3, 2, y_hi=out.hi, y_lo=out.lo, off_y=512))
        return out

    def _block_e(self, b, x, feats=None):
        n, h, w, _ = x.hi.shape
        raw, col = self._conv([b + ".branch1x1", b + ".branch3x3_1", b + ".branch3x3dbl_1", b + ".branch_pool"], x)
        ta, tb = Operands((n, h, w, 384), self.dev, SPLIT), Operands((n, h, w, 448), self.dev, SPLIT)
        self._seg(raw, col[b + ".branch3x3_1"], b + ".branch3x3_1", ta, 0)
        self._seg(raw, col[b + ".branch3x3dbl_1"], b + ".branch3x3dbl_1", tb, 0)
        tc = self._single(b + ".branch3x3dbl_2", tb)
        branches = ((ta, "branch3x3_2a", 320), (ta, "branch3x3_2b", 704), (tc, "branch3x3dbl_3a", 1088),
                    (tc, "branch3x3dbl_3b", 1472))
        if feats is None:
            out = Operands((n, h, w, 2048), self.dev, SPLIT)
            self._seg(raw, col[b + ".branch1x1"], b + ".branch1x1", out, 0)
            self._seg(raw, col[b + ".branch_pool"], b + ".branch_pool", out, 1856, box=True)
            for src, nm, off in branches:
                self._single(b + "." + nm, src, y=out, off=off)
            return out
        # Mixed_7c: every branch straight into the [N, 2048] features (torch.cat order 320 | 768 | 768 | 192)
        f1, fp = self._f32(n, h, w, 320), self._f32(n, h, w, 192)
        self._seg(raw, col[b + ".branch1x1"], b + ".branch1x1", None, 0, f32=f1)
        self._seg(raw, col[b + ".branch_pool"], b + ".branch_pool", None, 0, box=True, f32=fp)
        self.ops.append(lambda: K.global_avgpool_nhwc(f1, out=feats[:, 0:], ld_out=2048))
        for src, nm, off in branches:
            r, _ = self._conv([b + "." + nm], src)
            self._gap(r, b + "." + nm, off)
        self.ops.append(lambda: K.global_avgpool_nhwc(fp, out=feats[:, 1856:], ld_out=2048))

    def run(self, frames):
        """-> features [N, 2048] (a view valid until the next run)."""
        K.inception_input(frames, out=self.x)
        for op in self.ops:
            op()
        return self.feats


class InceptionFeatures(object):
    """InceptionV3(output_blocks=[3], resize_input=False, normalize_input=False) of his_evaluators behind the metric
    classes' preprocess: [N,3,H,W] frames in [0,1] -> [N, 2048] fp32 pool features on the device."""

    def __init__(self, device=None, weights=None):
        self.device = _device(device)
        convs = load_inception_weights(weights)
        # Conv2d_1a: BN folded into the fp32 direct stem (its output is the only one not on the conv engine)
        w, scale, shift = convs["Conv2d_1a_3x3"]
        self.stem_w = (w.double() * scale.double().view(-1, 1, 1, 1)).float().to(self.device).contiguous()
        self.stem_b = shift.to(self.device).contiguous()
        self.convs = convs

    def stream(self, n, h, w):
        return stream_for(self, _InceptionStream, (n, h, w), n, h, w, self.device, limit=2)

    def __call__(self, frames):
        """-> fresh [N, 2048] fp32 CUDA tensor."""
        x = _frames(frames, self.device)
        n, _, h, w = x.shape
        with torch.cuda.device(self.device):
            return self.stream(n, h, w).run(x).clone()


_INCEPTION = {}                                                      # metrics.py's MODEL_ZOOS: one network per device


def _shared_inception(device, weights):
    dev = _device(device)
    if weights is not None:
        return InceptionFeatures(dev, weights)
    if dev not in _INCEPTION:
        _INCEPTION[dev] = InceptionFeatures(dev)
    return _INCEPTION[dev]


def _f64(x, device=None):
    """numpy / tensor -> float64 tensor on ``device``; by default tensors stay where they are and numpy goes to the
    current CUDA device when there is one."""
    if torch.is_tensor(x):
        return x.to(device=device if device is not None else x.device, dtype=torch.float64)
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
    return torch.as_tensor(np.asarray(x)).to(device=device, dtype=torch.float64)


class _UnpairedScores(object):
    """The static score functions of BaseMetric (metrics.py:309-395) in float64 torch; numpy or tensors in, floats out."""

    @staticmethod
    def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
        """||mu1 - mu2||^2 + tr(s1) + tr(s2) - 2 tr sqrtm(s1 s2), with tr sqrtm(s1 s2) = sum sqrt(max(l, 0)) over the
        eigenvalues l of the symmetric s1^1/2 s2 s1^1/2 (similar to s1 s2).  Unlike the reference's scipy sqrtm, a
        rank-deficient product needs no eps retry and never has imaginary parts: the real trace is returned (``eps``
        is accepted for the reference's signature and unused)."""
        mu1 = _f64(mu1).reshape(-1)
        mu2 = _f64(mu2, mu1.device).reshape(-1)
        s1 = _f64(sigma1, mu1.device)
        s2 = _f64(sigma2, mu1.device)
        s1 = s1.reshape(1, 1) if s1.dim() < 2 else s1
        s2 = s2.reshape(1, 1) if s2.dim() < 2 else s2
        if mu1.shape != mu2.shape or s1.shape != s2.shape or s1.shape[0] != mu1.numel():
            raise LwbError("Frechet distance: means %s / %s and covariances %s / %s disagree"
                           % (tuple(mu1.shape), tuple(mu2.shape), tuple(s1.shape), tuple(s2.shape)))
        lam, v = torch.linalg.eigh(s1)
        r1 = (v * lam.clamp_min(0).sqrt()) @ v.T
        m = r1 @ s2 @ r1
        tr_covmean = torch.linalg.eigvalsh((m + m.T) * 0.5).clamp_min(0).sqrt().sum()
        diff = mu1 - mu2
        return float(diff @ diff + torch.trace(s1) + torch.trace(s2) - 2 * tr_covmean)

    @staticmethod
    def fid_score_func(pred_feats, gt_feats):
        """FID of two [N, D] feature sets: means and covariances (ddof=1, as np.cov) in float64.  An empty set scores
        0 as in the reference; a set of one frame raises (np.cov would give NaN)."""
        if len(pred_feats) == 0 or len(gt_feats) == 0:
            return 0.0
        a = _f64(pred_feats)
        b = _f64(gt_feats, a.device)
        if a.shape[0] < 2 or b.shape[0] < 2:
            raise LwbError("FID needs at least 2 frames per set (got %d and %d)" % (a.shape[0], b.shape[0]))
        stats = []
        for x in (a, b):
            mu = x.mean(0)
            xc = x - mu
            stats += [mu, xc.T @ xc / (x.shape[0] - 1)]
        return _UnpairedScores.calculate_frechet_distance(*stats)

    @staticmethod
    def is_score_func(feats_softmax):
        """exp(mean_i KL(p_i || mean_j p_j)) of softmax rows [N, K], in float64."""
        p = _f64(feats_softmax)
        kl = p * (torch.log(p) - torch.log(p.mean(0, keepdim=True)))
        return float(torch.exp(kl.sum(1).mean()))


class InceptionScoreMetric(_UnpairedScores):
    """metrics.py:634-701.  The shared model stops at block 3, so the softmax runs over the 2048 pool features, not
    over the 1000 ImageNet logits: the scores are comparable with the reference's, not with published Inception
    Scores."""

    def __init__(self, device=None, weights=None):
        self.device = _device(device)
        self.net = _shared_inception(self.device, weights)
        self.height, self.width = 299, 299

    def forward(self, imgs):
        """[N,3,H,W] frames in [0,1] -> numpy float32 softmax of the features [N, 2048]."""
        return torch.softmax(self.net(imgs), dim=1).cpu().numpy()

    def calculate_score(self, preds, batch_size=32):
        """(mean, std) of the per-``batch_size``-chunk scores; features stay on the device."""
        scores = []
        for i in range(int(math.ceil(len(preds) / batch_size))):
            f = self.net(preds[i * batch_size: (i + 1) * batch_size])
            scores.append(self.is_score_func(torch.softmax(f.double(), dim=1)))
        return float(np.mean(scores)), float(np.std(scores))

    def quality(self):
        return HIGHER


class FIDMetric(_UnpairedScores):
    """metrics.py:704-781."""

    def __init__(self, device=None, weights=None):
        self.device = _device(device)
        self.net = _shared_inception(self.device, weights)
        self.height, self.width = 299, 299

    def forward(self, imgs):
        """[N,3,H,W] frames in [0,1] -> numpy float32 features [N, 2048]."""
        return self.net(imgs).cpu().numpy()

    def calculate_score(self, preds, gts, batch_size=32):
        """FID of the features of all preds against all gts (chunks of ``batch_size``), kept on the device."""
        pf, gf = [], []
        for i in range(int(math.ceil(len(preds) / batch_size))):
            pf.append(self.net(preds[i * batch_size: (i + 1) * batch_size]))
            gf.append(self.net(gts[i * batch_size: (i + 1) * batch_size]))
        if not pf:
            return self.fid_score_func([], [])
        return self.fid_score_func(torch.cat(pf), torch.cat(gf))

    def quality(self):
        return LOWER
