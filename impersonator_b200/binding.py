"""Host-side binding of the networks that run on the conv engine (the generator, HMR, the inpaintor, the Mask R-CNN
detector, LPIPS' AlexNet and InceptionV3): operand buffers, the operand mode, weight packing with one host sync per
network, conv plans, eval-mode BatchNorm folding and the per-shape stream caches.  Every kernel call goes through the
``kernels`` module, so that tests can substitute its front-ends."""
import os

import torch

from . import graph as _graph
from . import kernels as K
from ._lib import LwbError

DEFAULT_PRECISION = "fp16f8"

# Bits of the operand-range flag (LWB_RANGE_* of include/lwb_b200.h)
RANGE_F8 = 1            # an emitted operand has |x| >= 1024: its e4m3 correction terms clip
RANGE_FP16 = 2          # |x| >= 60000 or not finite: the fp16 hi itself overflows
RANGE_HEADS = 4         # a head pre-activation reached +-8


def precision_mode():
    return os.environ.get("LWB_PRECISION", DEFAULT_PRECISION)


def split_mode(mod=None):
    """LWB_PRECISION (or the module's set_precision pin) -> operand split code of the conv engine (lwb_conv_desc.split):
    fp16x3 = 1: x_hi*w_hi + x_hi*w_lo + x_lo*w_hi, all fp16 (3 MMAs per K step);
    fp16f8 = 2: x_hi*w_hi in fp16 + (x*w_lo, x_lo*w) in e4m3 at twice the rate (2 MMA-equivalents per K step);
    fp16   = 0: single pass (not parity-gated)."""
    mode = (getattr(mod, '_lwb_precision', None) if mod is not None else None) or precision_mode()
    codes = {"fp16": 0, "fp16x3": 1, "fp16f8": 2}
    if mode not in codes:
        raise LwbError("LWB_PRECISION must be fp16x3, fp16f8 or fp16")
    return codes[mode]


def lo_format(split):
    """The lo operand format the epilogues emit for conv plans of operand mode ``split``: 1 (fp8 pair blocks) for
    fp16f8, else 0 (fp16)."""
    return 1 if split == 2 else 0


class Operands(object):
    """An NHWC activation: fp16 hi / lo operands of the next conv (lo only when split != 0; none with half=False) and an
    optional fp32 copy."""
    __slots__ = ("hi", "lo", "f32")

    def __init__(self, shape, dev, split=1, f32=False, half=True):
        self.hi = torch.empty(shape, dtype=torch.float16, device=dev) if half else None
        self.lo = torch.empty(shape, dtype=torch.float16, device=dev) if (half and split) else None
        self.f32 = torch.empty(shape, dtype=torch.float32, device=dev) if f32 else None

    @property
    def pair(self):
        """(hi, lo), the operand argument of K.ConvPlan."""
        return (self.hi, self.lo)

    def out(self):
        """The output keywords of the epilogue front-ends."""
        return dict(y_f32=self.f32, y_hi=self.hi, y_lo=self.lo)


def _convt_merge():
    """LWB_CONVT_MERGE (default 1): ConvTranspose2d(k3, s2, p1, op1) layers with up to 128 output channels run as ONE
    stride-1 pass with the four sub-pixel phases stacked on N (merge_transposed_weight) instead of four phase launches."""
    return os.environ.get("LWB_CONVT_MERGE", "1") != "0"


def merge_transposed_weight(wt):
    """IOHW [cin, cout, 3, 3] of ConvTranspose2d(k=3, s=2, p=1, output_padding=1) -> OIHW [4*cout, cin, 2, 2]: output
    channel block ph = 2a + b holds sub-pixel phase out[2y+a, 2x+b]; filter tap (dy, dx) reads in[y+dy, x+dx].
    Per axis: phase 0 uses k=1 at d=0; phase 1 uses k=2 at d=0 and k=0 at d=1 (oy = 2*iy - 1 + ky); the other 7 of the 16
    (phase, tap) blocks are zero."""
    cin, cout = wt.shape[0], wt.shape[1]
    k_of = ({0: 1}, {0: 2, 1: 0})
    out = torch.zeros((4 * cout, cin, 2, 2), dtype=torch.float32, device=wt.device)
    for a in range(2):
        for b in range(2):
            ph = 2 * a + b
            for dy, ky in k_of[a].items():
                for dx, kx in k_of[b].items():
                    out[ph * cout:(ph + 1) * cout, :, dy, dx] = wt[:, :, ky, kx].t().float()
    return out


class Conv(object):
    """One convolution bound to its operands: ``desc``, the raw fp32 NHWC output ``out`` and, after
    PlanBinder.finalize(), ``plan``."""
    __slots__ = ("desc", "x", "x1", "weight", "cout_pad", "cin_pad", "stats", "out", "plan")


class PlanBinder(object):
    """Collects the convolutions of one stream, then packs every weight with one host sync and creates the plans."""

    def __init__(self, dev, split):
        self.dev, self.split = dev, split
        self._shared = {}
        self._convs = []

    def conv(self, weight, x, n, h, w, stride=1, pad=None, pad_w=None, dil=1, cout_pad=None, cin_pad=None, out=None,
             share=None, x1=None, transposed=False, rowk=False, row_pitch=0, n_tile=0, halo=False, split=None,
             stats=None):
        """weight OIHW fp32 over operands x = (hi, lo) of [n, h, w, cin_pad or cin]; pad defaults to kh // 2.  The raw
        output [n, ho, wo, cout_pad or cout] is ``out`` when given, else the buffer shared by every conv of this binder
        with the same output shape and ``share`` tag when one is given, else a buffer of its own.
        x1: second operand pair of a concat input, its channels follow those of x.  transposed: IOHW weights of a
        ConvTranspose2d(k3, s2, p1, op1), run as one merged-phase pass (lwb_conv_desc.transposed = 2) where
        LWB_CONVT_MERGE and the shape allow.  rowk: the 7x7 row-K stem over rows of ``row_pitch`` pixels of cin_pad
        channels.  n_tile / halo: lwb_conv_desc's forced N tile and halo variant.  split: this conv's operand mode (the
        binder's by default).  stats: f64 [n, cout, 2] InstanceNorm sums the plan accumulates."""
        cout, cin = (weight.shape[1], weight.shape[0]) if transposed else (weight.shape[0], weight.shape[1])
        kh, kw = weight.shape[2:]
        cin1 = x1[0].shape[3] if x1 is not None else 0
        r = Conv()
        r.desc = K.make_conv_desc(n, h, w, (cin_pad or cin) - cin1, cout_pad or cout, kh, kw, stride=stride,
                                  pad=kh // 2 if pad is None else pad, pad_w=pad_w, dil=dil, cin1=cin1,
                                  transposed=transposed, split=self.split if split is None else split, rowk=rowk,
                                  row_pitch=row_pitch, n_tile=n_tile, halo=halo)
        if transposed and _convt_merge() and cout <= 128 and cout % 32 == 0 and (kh, kw) == (3, 3):
            r.desc.transposed = 2
            weight = merge_transposed_weight(weight)
        shape = (n, r.desc.h_out, r.desc.w_out, cout_pad or cout)
        if out is None and share is not None:
            out = self._shared.get((shape, share))
            if out is None:
                out = self._shared[(shape, share)] = torch.empty(shape, dtype=torch.float32, device=self.dev)
        r.out = out if out is not None else torch.empty(shape, dtype=torch.float32, device=self.dev)
        r.x, r.x1, r.weight, r.cout_pad, r.cin_pad, r.stats, r.plan = x, x1, weight, cout_pad, cin_pad, stats, None
        self._convs.append(r)
        return r

    def finalize(self):
        """Pack the weights and create every K.ConvPlan; the fp32 source weights are released.  max|w| of every layer
        is read back in ONE host sync (it sets the per-layer weight exponent, kernels.weight_exponent)."""
        convs, self._convs = self._convs, []
        amax = torch.stack([r.weight.abs().max().float() for r in convs]).tolist()
        packed = [K.pack_conv_weight_rowk(r.weight, cout_pad=r.cout_pad, cpx=r.cin_pad, split=r.desc.split, absmax=a)
                  if r.desc.rowk else
                  K.pack_conv_weight(r.weight, transposed=r.desc.transposed == 1, cout_pad=r.cout_pad, cin_pad=r.cin_pad,
                                     split=r.desc.split, absmax=a)
                  for r, a in zip(convs, amax)]
        for r, wp in zip(convs, packed):
            r.plan = K.ConvPlan(r.desc, r.x, r.x1, wp, r.out, r.stats)
            r.weight = None


def stream_for(owner, cls, key, *args, limit, **kw):
    """The per-shape stream ``cls(owner, *args, **kw)`` cached under ``key`` in ``owner.__dict__['_lwb_streams']``: the
    ``limit`` most recently used shapes are kept (each holds its activations, plans and packed weights)."""
    streams = owner.__dict__.setdefault('_lwb_streams', {})
    if key in streams:
        streams[key] = streams.pop(key)                  # most recently used last
    else:
        while len(streams) >= limit:
            streams.pop(next(iter(streams)))
        streams[key] = cls(owner, *args, **kw)
    return _graph.pin(streams[key])                      # a CUDA graph being captured keeps what it replays into alive


class StreamOwner(object):
    """Mixin of the nn.Modules that cache streams with stream_for: loading parameters or moving / casting the module
    (``_apply``) drops them, so the next call rebuilds them from the current weights."""

    def _lwb_invalidate(self):
        self.__dict__['_lwb_streams'] = {}

    def load_state_dict(self, *args, **kwargs):
        out = super(StreamOwner, self).load_state_dict(*args, **kwargs)
        self._lwb_invalidate()
        return out

    def _apply(self, fn, *args, **kwargs):
        out = super(StreamOwner, self)._apply(fn, *args, **kwargs)
        self._lwb_invalidate()
        return out


def bn_affine(weight, bias, mean, var, eps):
    """Eval-mode BatchNorm as y = x * scale + shift: folded in float64, returned as contiguous fp32 (scale, shift)."""
    scale = weight.detach().double() / torch.sqrt(var.detach().double() + eps)
    shift = bias.detach().double() - mean.detach().double() * scale
    return scale.float().contiguous(), shift.float().contiguous()
