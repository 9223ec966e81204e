"""Host-side mirror of networks/generator.py (the reference's generator), running on the
hand-written sm_90a conv engine behind the C ABI.

Same class names, constructor arguments, method signatures and ``state_dict`` keys as the
reference, so checkpoints (``BaseModel._load_params``, models/models.py:159-179) and callers
(models/imitator.py, swapper.py, viewer.py) work unchanged:

  ResidualBlock            networks/generator.py:8-20
  ResNetGenerator          networks/generator.py:23-65     (BG net)
  ResUnetGenerator         networks/generator.py:68-184    (SID / TSF nets)
  ImpersonatorGenerator    networks/generator.py:187-320   (forward, encode_src, infer_front, swap,
                                                            inference, resize_trans, stn, transform)

The ``nn.Conv2d`` / ``nn.InstanceNorm2d`` / ``nn.ConvTranspose2d`` children are parameter holders
only (they give the reference's key names and default init); every forward path goes through
``_Stream`` below, which drive hand-written sm_90a kernels:
wgmma implicit-GEMM convs (fp16 hi/lo split operands, fp32 accumulate), a fused
InstanceNorm+ReLU+residual+Liquid-Warping-Block kernel, and the 7x7 heads.  There is no torch
fallback: without the CUDA library the calls raise.

Extensions over the reference (all optional): source features may have batch 1 while the target
batch is B (torch's grid_sample cannot broadcast); ``LWB_PRECISION=fp16`` selects the
single-pass "fast" mode (the default ``fp16f8`` and ``fp16x3`` both meet the 1e-3 parity bar, see binding.split_mode);
the LWB's grid_sample follows the reference's pinned torch 1.2 (align_corners=True), ``LWB_ALIGN_CORNERS=0``
selects what torch >= 1.3 does for the same flag-less call (kernels.default_align_corners).
"""
import os

import torch
import torch.nn as nn

from . import kernels as K
from ._lib import LwbError
from .binding import Operands, PlanBinder, StreamOwner, lo_format, precision_mode, split_mode, stream_for
from .binding import merge_transposed_weight  # noqa: F401  (callers import it from the generator too)


_WEIGHTS_EPOCH = [0]
_PASS = [0]                                              # bumped by every ImpersonatorGenerator entry point; streams stamp it


def _new_pass():
    _PASS[0] += 1



def weights_epoch():
    """Bumped whenever a network's parameters may have changed (load_state_dict, init_weights, .to()/.half()...): packed
    weights and per-shape streams are rebuilt then, and anything that cached launches against them must be rebuilt too."""
    return _WEIGHTS_EPOCH[0]


def _sub_batches(B, enc_w, res_w, bg):
    """LWB_STREAMS (default 2, at most 2): number of concurrent sub-batches ImpersonatorGenerator.inference splits a batch
    into.  Only when the source features / background are shared by the batch (the imitation case), B divides evenly and
    every sub-batch keeps at least 4 frames."""
    try:
        n = min(2, int(os.environ.get("LWB_STREAMS", "2")))
    except ValueError:
        n = 1
    if n <= 1 or B % n or B // n < 4:
        return 1
    shared = all(t is None or t.shape[0] == 1 for t in list(enc_w) + list(res_w)) and (bg is None or bg.shape[0] == 1)
    return n if shared else 1


def _tc_heads():
    """LWB_TC_HEADS (default 1): the 7x7 output heads run on the tensor cores as a 7x1 filter whose N dimension
    carries the 7 filter columns x 4 head channels (28 -> 32); the composite kernel sums the columns.  0 = the fp32
    CUDA-core kernel (k_heads7x7)."""
    return os.environ.get("LWB_TC_HEADS", "1") != "0"


def fold_head_weights(w_img, w_att):
    """[3,64,7,7] + [1,64,7,7] -> [32, 64, 7, 1]: output channel kx*4 + co of the (7 x 1) filter = column kx of head co
    (networks/generator.py:126-134; rows 28..31 are zero)."""
    w4 = torch.cat([w_img, w_att], dim=0).float()                      # [4, C, ky, kx]
    folded = w4.permute(3, 0, 1, 2).reshape(28, w4.shape[1], 7, 1)     # [kx*4+co, C, ky, 1]
    return torch.cat([folded, torch.zeros(4, w4.shape[1], 7, 1, dtype=folded.dtype, device=folded.device)], dim=0).contiguous()


STEM_MAX_CIN = 24                                          # input channels the row-K stem takes (3 + the widest map, 15)


def stem_cin_pad(cin):
    """Channels per pixel of the stem's padded input for ``cin`` input channels: 8 (one K stage of 64 per filter row),
    16 or 24 (two or three stages): the 3 + cond channels of every map of mesh.get_map_fn_dim fit."""
    if not 0 < cin <= STEM_MAX_CIN:
        raise LwbError("the 7x7 stem takes 1 to %d input channels, not %d" % (STEM_MAX_CIN, cin))
    return (cin + 7) // 8 * 8


def _halo_mode():
    """LWB_HALO: '0' (default) = CUDA-core 7x7 heads; 'auto' = halo plans for the row-K stem and the skippers + 7x7
    heads on tensor cores (N tile 16); 'all' = also the residual blocks.  Halo plans run through the same tap-group conv
    kernel as the others."""
    if precision_mode() == "fp16f8":
        return '0'                                         # halo plans have no fp8 path
    return os.environ.get("LWB_HALO", "0")


class NetworkBase(StreamOwner, nn.Module):
    """networks/networks.py:45-80."""

    def __init__(self):
        super(NetworkBase, self).__init__()
        self._name = 'BaseNetwork'

    @property
    def name(self):
        return self._name

    def init_weights(self):
        self.apply(self._weights_init_fn)
        self._lwb_invalidate()

    def _weights_init_fn(self, m):
        classname = m.__class__.__name__
        if classname.find('Conv') != -1:
            m.weight.data.normal_(0.0, 0.02)
            if hasattr(m.bias, 'data'):
                m.bias.data.fill_(0)
        elif classname.find('BatchNorm2d') != -1:
            m.weight.data.normal_(1.0, 0.02)
            m.bias.data.fill_(0)

    def _lwb_invalidate(self):
        _WEIGHTS_EPOCH[0] += 1                               # captured graphs keyed on it (imitator._chunk_step) are re-captured
        for m in self.modules():
            if hasattr(m, '_lwb_streams'):
                m._lwb_streams = {}

    def set_precision(self, mode):
        """Pin this network (and its sub-networks) to an operand mode regardless of LWB_PRECISION (None = follow the env)."""
        if mode not in (None, "fp16", "fp16x3", "fp16f8"):
            raise LwbError("precision must be fp16x3, fp16f8, fp16 or None")
        for m in self.modules():
            if isinstance(m, NetworkBase):
                m.__dict__['_lwb_precision'] = mode

    def range_flags(self):
        """-> list of int32[1] device tensors, one per stream used by the most recent pass, with the bits
        binding.RANGE_F8 = an activation left the e4m3 correction range (|x| >= 1024, fp16f8 precision degrades for those
        elements), binding.RANGE_FP16 = the fp16 range (|x| >= 60000 / NaN), binding.RANGE_HEADS = output-head
        pre-activations of +-8 and more in fp16f8 mode (its ~1e-4 relative end-to-end precision then no longer guarantees
        1e-3 on the pixels: use fp16x3)."""
        live = []
        for m in self.modules():
            for st in getattr(m, '_lwb_streams', {}).values():
                live.append((getattr(st, 'pass_id', -1), st.range_flag))
        if not live:
            return []
        last = max(p for p, _ in live)                       # streams of other shapes / precisions keep the bits of older passes
        return [f for p, f in live if p == last]

    def range_flag_tensor(self):
        """One int32 device scalar = OR over the live streams' flags; None if no stream exists yet.  No host sync."""
        flags = self.range_flags()
        if not flags:
            return None
        if len(flags) == 1:
            return flags[0]
        acc = flags[0].clone()
        for f in flags[1:]:
            acc |= f
        return acc

    def range_status(self):
        """OR of range_flags() as a Python int (one device sync); streams reset their flag at the start of a pass."""
        flags = self.range_flags()
        if not flags:
            return 0
        bits = torch.stack([f.reshape(()) for f in flags]).cpu()
        out = 0
        for b in bits.tolist():
            out |= int(b)
        return out



class ResidualBlock(nn.Module):
    """networks/generator.py:8-20 (parameter holder)."""

    def __init__(self, dim_in, dim_out):
        super(ResidualBlock, self).__init__()
        self.main = nn.Sequential(
            nn.Conv2d(dim_in, dim_out, kernel_size=3, stride=1, padding=1, bias=False),
            nn.InstanceNorm2d(dim_out, affine=True),
            nn.ReLU(inplace=True),
            nn.Conv2d(dim_out, dim_out, kernel_size=3, stride=1, padding=1, bias=False),
            nn.InstanceNorm2d(dim_out, affine=True))

    def forward(self, x):
        raise LwbError("ResidualBlock runs only inside the fused generator streams")


# ------------------------------------------------------------------------------------------
# engine: one network bound to (batch, H, W, precision) -> persistent buffers + conv plans
# ------------------------------------------------------------------------------------------
class _Stream(object):
    """ResUnetGenerator (networks/generator.py:68-184) or ResNetGenerator (networks/generator.py:23-65, the BG net: the
    same chain without skippers and warps) bound to fixed shapes."""

    def __init__(self, net, B, H, W, dev, split, keep_f32=False):
        self.B, self.H, self.W, self.split = B, H, W, split
        if isinstance(net, ResUnetGenerator):
            enc, dec, skip = ([(s[0], s[1]) for s in seq] for seq in (net.encoders, net.decoders, net.skippers))
            blocks = [b.main for b in net.resnets]
            w_img, w_att = net.img_reg[0].weight.detach(), net.attetion_reg[0].weight.detach()
        else:                                                     # the BG net: one flat Sequential, a 3-channel head
            m, r = list(net.model), 3 * (net._n_down + 1)
            enc = [(m[i], m[i + 1]) for i in range(0, r, 3)]
            blocks = [b.main for b in m[r:r + net._repeat_num]]
            dec = [(m[i], m[i + 1]) for i in range(r + net._repeat_num, len(m) - 2, 3)]
            skip = []
            w_img = m[-2].weight.detach()
            w_att = torch.zeros_like(w_img[:1])
        self.n_down = nd = len(dec)
        if H % (1 << nd) or W % (1 << nd):
            raise LwbError("image size must be divisible by %d" % (1 << nd))
        self.cin = enc[0][0].weight.shape[1]
        self.cin_pad = stem_cin_pad(self.cin)
        # InstanceNorm statistics of every conv + the operand-range flag share one buffer: one fill per pass
        norms = [m for m in net.modules() if isinstance(m, nn.InstanceNorm2d)]
        cmax = max([16] + [m.num_features for m in norms])
        nstat = len(norms) * B * cmax * 2
        self._zero = torch.zeros(nstat * 8 + 4, dtype=torch.uint8, device=dev)
        slots = iter(self._zero[:nstat * 8].view(torch.float64).view(len(norms), -1))
        self.range_flag = self._zero[nstat * 8:].view(torch.int32)
        self.ws = torch.empty((B, cmax, 2), dtype=torch.float32, device=dev)
        plans = PlanBinder(dev, split)

        def conv_norm(conv, norm, x, h, w, **kw):
            """-> (Conv, gamma, beta); the conv accumulates its statistics in the next slot (a contiguous [B, cout, 2]
            view at its head)."""
            c = norm.num_features
            stats = next(slots)[:B * c * 2].view(B, c, 2)
            return (plans.conv(conv.weight.detach(), x, B, h, w, share="raw", stats=stats, **kw),
                    norm.weight.detach().float().contiguous(), norm.bias.detach().float().contiguous())

        hm = _halo_mode() if skip else '0'                        # the BG net ignores LWB_HALO
        c0 = enc[0][0].weight.shape[0]
        tc = _tc_heads() and c0 == 64                            # folded heads, unless the halo heads run
        heads_tc = hm != '0' or tc                                # the heads read fp16 operands, else fp32
        # stem input: padded NHWC of 8, 16 or 24 channels (3 px border top/left/bottom, 5 right) for the row-K 7x7 conv,
        # which keeps the fp16 hi/lo input
        self.x_pad = Operands((B, H + 6, W + 8, self.cin_pad), dev, split)
        self.enc_layers = [conv_norm(*enc[0], self.x_pad.pair, H, W, rowk=True, row_pitch=W + 8, cin_pad=self.cin_pad,
                                     split=min(split, 1), halo=(hm != '0'))]
        c, h, w = c0, H, W
        self.e = [Operands((B, h, w, c), dev, split, f32=keep_f32)]
        for i in range(1, nd + 1):
            self.enc_layers.append(conv_norm(*enc[i], self.e[i - 1].pair, h, w, stride=2))
            c, h, w = c * 2, h // 2, w // 2
            self.e.append(Operands((B, h, w, c), dev, split, f32=(keep_f32 or i == nd)))
        # resnets (h buffer for the mid activation)
        self.hb = Operands((B, h, w, c), dev, split)
        self.res_layers, self.res_out = [], []
        prev = self.e[nd]
        for m in blocks:
            self.res_layers.append((conv_norm(m[0], m[1], prev.pair, h, w, halo=(hm == 'all')),
                                    conv_norm(m[3], m[4], self.hb.pair, h, w, halo=(hm == 'all'))))
            prev = Operands((B, h, w, c), dev, split, f32=True)
            self.res_out.append(prev)
        # decoders, each followed by its skipper (concat input: encoder output, decoder output) where the net has them
        self.dec_layers, self.d_up, self.d_out = [], [], []
        for i, (conv, norm) in enumerate(dec):
            last = (i == nd - 1)
            out = Operands((B, h * 2, w * 2, c // 2), dev, split, f32=(last and not heads_tc), half=(not last or heads_tc))
            up = Operands((B, h * 2, w * 2, c // 2), dev, split) if skip else out
            ld = conv_norm(conv, norm, prev.pair, h, w, stride=2, transposed=True)
            c, h, w = c // 2, h * 2, w * 2
            ls = conv_norm(*skip[i], self.e[nd - 1 - i].pair, h, w, x1=up.pair, halo=(hm != '0')) if skip else None
            self.dec_layers.append((ld, ls))
            self.d_up.append(up)
            self.d_out.append(out)
            prev = out
        # img_reg (64->3) + attetion_reg (64->1)
        self.head, self.folded_kw = None, 0
        if hm != '0':
            # one 7x7 conv padded to 16 output channels on the tensor cores (halo variant, N tile 16); channels 0..3
            # are consumed by the composite kernel
            w16 = torch.cat([w_img, w_att, torch.zeros(12, *w_img.shape[1:], device=w_img.device, dtype=w_img.dtype)], dim=0)
            self.head = plans.conv(w16, prev.pair, B, H, W, halo=True, n_tile=16, share="raw")
        elif tc:
            # a 7 x 1 filter with N = 7 columns x 4 channels (-> 32) on the tensor cores; the composite kernel adds the
            # seven column partials of every pixel (lwb_heads_composite, folded_kw)
            self.head = plans.conv(fold_head_weights(w_img, w_att), prev.pair, B, H, W, pad_w=0, n_tile=32, share="raw")
            self.folded_kw = 7
        else:
            self.w4 = K.pack_head_weights(w_img, w_att)
            self.head_raw = torch.empty((B, H, W, 4), dtype=torch.float32, device=dev)
        plans.finalize()
        if self.head is not None:
            self.head_raw = self.head.out
        if self.folded_kw:
            # the folded heads issue N = 32 columns; their algorithmic work is the 7x7 x 64 -> 4 convolution
            p = self.head.plan
            p.flops = 2.0 * B * H * W * 49 * 64 * 4
            p.label = "H7x7 64->4 @%d (7x1 filter, N = 7 cols x 4)" % H
            p.prof_class = "heads"
        self.head_flag = self.range_flag if split == 2 and skip else None     # the BG net's heads report no range bit

    def begin_pass(self):
        """Zero the InstanceNorm statistics and the range flag (one fill)."""
        self._zero.zero_()
        self.pass_id = _PASS[0]

    def _conv_norm(self, layer, out, relu, residual=None, warp_src=None, T=None, ac=False):
        conv, gamma, beta = layer
        conv.plan.run()
        K.norm_act_nhwc(conv.out, conv.stats, gamma, beta, relu, self.ws, residual=residual, warp_src=warp_src, T=T,
                        align_corners=ac, y_f32=out.f32, y_hi=out.hi, y_lo=out.lo, lo_format=lo_format(self.split),
                        range_flag=self.range_flag)

    # ---- pieces -------------------------------------------------------------------------
    def load_input(self, x):
        if tuple(x.shape) != (self.B, self.cin, self.H, self.W) or x.dtype != torch.float32:
            raise LwbError("unexpected input %s (stream built for %s)" % (tuple(x.shape), (self.B, self.cin, self.H, self.W)))
        K.nchw_to_nhwc_split(x.contiguous(), c_pad=self.cin_pad, pad_hw=(3, 3, 3, 5), hi=self.x_pad.hi, lo=self.x_pad.lo)

    def encode(self, warp_srcs=None, T=None, ac=False):
        """encoders 0..n_down; warp_srcs[i] (NHWC fp32, i >= 1) is LWB-added after encoder i."""
        self.begin_pass()
        self._conv_norm(self.enc_layers[0], self.e[0], True)
        for i in range(1, self.n_down + 1):
            src = warp_srcs[i] if warp_srcs is not None else None
            if isinstance(src, (list, tuple)):          # swap(): two warps per site
                self._conv_norm(self.enc_layers[i], self.e[i], True, warp_src=src[0][0], T=src[0][1], ac=ac)
                self._add_warp(self.e[i], src[1][0], src[1][1], ac)
            else:
                self._conv_norm(self.enc_layers[i], self.e[i], True, warp_src=src, T=T, ac=ac)

    def _add_warp(self, act, src, T, ac):
        if act.f32 is None:
            raise LwbError("second warp needs an fp32 activation")
        K.norm_act_nhwc(act.f32, None, None, None, False, self.ws, warp_src=src, T=T, align_corners=ac,
                        y_f32=act.f32, y_hi=act.hi, y_lo=act.lo, lo_format=lo_format(self.split),
                        range_flag=self.range_flag)

    def resnets(self, warp_srcs=None, T=None, ac=False):
        x = self.e[self.n_down]
        for i, (l1, l2) in enumerate(self.res_layers):
            self._conv_norm(l1, self.hb, True)
            src = warp_srcs[i] if warp_srcs is not None else None
            if isinstance(src, (list, tuple)):
                self._conv_norm(l2, self.res_out[i], False, residual=x.f32, warp_src=src[0][0], T=src[0][1], ac=ac)
                self._add_warp(self.res_out[i], src[1][0], src[1][1], ac)
            else:
                self._conv_norm(l2, self.res_out[i], False, residual=x.f32, warp_src=src, T=T, ac=ac)
            x = self.res_out[i]

    def decode(self):
        for (ld, ls), up, out in zip(self.dec_layers, self.d_up, self.d_out):
            self._conv_norm(ld, up, True)
            if ls is not None:
                self._conv_norm(ls, out, True)

    def heads(self, bg=None, want_color=True, want_mask=True, **out):
        if self.head is not None:
            self.head.plan.run()
        else:
            K.conv7x7_heads_nhwc(self.d_out[-1].f32, self.w4, out=self.head_raw)
        return K.heads_composite(self.head_raw, bg, want_color=want_color, want_mask=want_mask, folded_kw=self.folded_kw,
                                 range_flag=self.head_flag, **out)


def profile_streams(warm_fn, run_fn):
    """Instrumented passes: CUDA events around every kernel class (bench.py roofline / breakdown).
    -> {"passes": n, "conv": {"ms", "flops", "n"}, "norm": {"ms", "bytes", "n"}, "heads"/"correspond"/"input": {"ms", ...}}"""
    warm_fn()
    torch.cuda.synchronize()
    K.profile_begin()
    n = len(run_fn())
    raw = K.profile_end()
    out = {"passes": n}
    for cls in ("conv", "norm", "heads", "correspond", "input"):
        r = raw.get(cls, {"ms": 0.0, "work": 0.0, "n": 0})
        out[cls] = {"ms": r["ms"], "n": r["n"], ("flops" if cls in ("conv", "heads") else "bytes"): r["work"]}
    out["layers"] = {k: {"ms": v["ms"] / n, "n": v["n"] / n, "work": v["work"] / n} for k, v in raw.items() if "/" in k}
    return out


def _stream_for(mod, cls, key, *args, **kw):
    """The generator networks' per-shape stream cache: the 8 most recently used shapes (each holds ~GBs at B=16)."""
    return stream_for(mod, cls, key, *args, limit=8, **kw)


def _nhwc_of(t):
    """NHWC fp32 twin of an NCHW feature (cached on the tensor by encode_src / inference)."""
    cached = getattr(t, '_lwb_nhwc', None)
    if cached is not None:
        return cached
    return t.permute(0, 2, 3, 1).contiguous()


def _nchw_outs(acts):
    """NCHW copies of the fp32 activations, each carrying its NHWC twin for _nhwc_of."""
    outs = []
    for a in acts:
        t = K.nhwc_to_nchw(a.f32)
        t._lwb_nhwc = a.f32.clone()
        outs.append(t)
    return outs


class ResNetGenerator(NetworkBase):
    """Generator. Encoder-Decoder Architecture (networks/generator.py:23-65)."""

    def __init__(self, conv_dim=64, c_dim=5, repeat_num=9, k_size=4, n_down=2):
        super(ResNetGenerator, self).__init__()
        self._name = 'resnet_generator'
        self._n_down, self._repeat_num = n_down, repeat_num
        if k_size != 3:
            raise LwbError("the conv engine implements k_size=3 (what ImpersonatorGenerator uses)")
        layers = []
        layers.append(nn.Conv2d(c_dim, conv_dim, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.InstanceNorm2d(conv_dim, affine=True))
        layers.append(nn.ReLU(inplace=True))
        curr_dim = conv_dim
        for i in range(n_down):
            layers.append(nn.Conv2d(curr_dim, curr_dim * 2, kernel_size=k_size, stride=2, padding=1, bias=False))
            layers.append(nn.InstanceNorm2d(curr_dim * 2, affine=True))
            layers.append(nn.ReLU(inplace=True))
            curr_dim = curr_dim * 2
        for i in range(repeat_num):
            layers.append(ResidualBlock(dim_in=curr_dim, dim_out=curr_dim))
        for i in range(n_down):
            layers.append(nn.ConvTranspose2d(curr_dim, curr_dim // 2, kernel_size=k_size, stride=2, padding=1,
                                             output_padding=1, bias=False))
            layers.append(nn.InstanceNorm2d(curr_dim // 2, affine=True))
            layers.append(nn.ReLU(inplace=True))
            curr_dim = curr_dim // 2
        layers.append(nn.Conv2d(curr_dim, 3, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.Tanh())
        self.model = nn.Sequential(*layers)

    @torch.no_grad()
    def forward(self, x, c=None):
        if c is not None:
            c = c.unsqueeze(2).unsqueeze(3)
            c = c.expand(c.size(0), c.size(1), x.size(2), x.size(3))
            x = torch.cat([x, c], dim=1)
        B, _, H, W = x.shape
        split = split_mode(self)
        st = _stream_for(self, _Stream, ('bg', B, H, W, split), B, H, W, x.device, split)
        st.load_input(x.float())
        st.encode()
        st.resnets()
        st.decode()
        return st.heads(want_mask=False)[0]


class ResUnetGenerator(NetworkBase):
    """Generator. Encoder-Decoder Architecture (networks/generator.py:68-184)."""

    def __init__(self, conv_dim=64, c_dim=5, repeat_num=6, k_size=4, n_down=2):
        super(ResUnetGenerator, self).__init__()
        self._name = 'resunet_generator'
        self.repeat_num = repeat_num
        self.n_down = n_down
        if k_size != 3:
            raise LwbError("the conv engine implements k_size=3 (what ImpersonatorGenerator uses)")
        encoders = []
        encoders.append(nn.Sequential(
            nn.Conv2d(c_dim, conv_dim, kernel_size=7, stride=1, padding=3, bias=False),
            nn.InstanceNorm2d(conv_dim, affine=True),
            nn.ReLU(inplace=True)))
        curr_dim = conv_dim
        for i in range(n_down):
            encoders.append(nn.Sequential(
                nn.Conv2d(curr_dim, curr_dim * 2, kernel_size=k_size, stride=2, padding=1, bias=False),
                nn.InstanceNorm2d(curr_dim * 2, affine=True),
                nn.ReLU(inplace=True)))
            curr_dim = curr_dim * 2
        self.encoders = nn.Sequential(*encoders)
        resnets = []
        for i in range(repeat_num):
            resnets.append(ResidualBlock(dim_in=curr_dim, dim_out=curr_dim))
        self.resnets = nn.Sequential(*resnets)
        decoders, skippers = [], []
        for i in range(n_down):
            decoders.append(nn.Sequential(
                nn.ConvTranspose2d(curr_dim, curr_dim // 2, kernel_size=k_size, stride=2, padding=1, output_padding=1, bias=False),
                nn.InstanceNorm2d(curr_dim // 2, affine=True),
                nn.ReLU(inplace=True)))
            skippers.append(nn.Sequential(
                nn.Conv2d(curr_dim, curr_dim // 2, kernel_size=k_size, stride=1, padding=1, bias=False),
                nn.InstanceNorm2d(curr_dim // 2, affine=True),
                nn.ReLU(inplace=True)))
            curr_dim = curr_dim // 2
        self.decoders = nn.Sequential(*decoders)
        self.skippers = nn.Sequential(*skippers)
        layers = []
        layers.append(nn.Conv2d(curr_dim, 3, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.Tanh())
        self.img_reg = nn.Sequential(*layers)
        layers = []
        layers.append(nn.Conv2d(curr_dim, 1, kernel_size=7, stride=1, padding=3, bias=False))
        layers.append(nn.Sigmoid())
        self.attetion_reg = nn.Sequential(*layers)

    def _stream(self, x, keep_f32, tag):
        B, _, H, W = x.shape
        split = split_mode(self)
        return _stream_for(self, _Stream, (tag, B, H, W, split, keep_f32), B, H, W, x.device, split, keep_f32=keep_f32)

    @torch.no_grad()
    def inference(self, x):
        """encoder_outs [4], resnet_outs [6] as NCHW fp32 (networks/generator.py:136-147)."""
        st = self._stream(x, True, 'inference')
        st.load_input(x.float())
        st.encode()
        st.resnets()
        return _nchw_outs(st.e), _nchw_outs(st.res_out)

    @torch.no_grad()
    def forward(self, x):
        st = self._stream(x, False, 'forward')
        st.load_input(x.float())
        st.encode()
        st.resnets()
        st.decode()
        color, mask, _ = st.heads()
        return color, mask

    def encode(self, x):
        return self.inference(x)[0]

    def decode(self, x, encoder_outs):
        raise LwbError("decode() on detached tensors is not part of the inference hot path; use forward()/inference()")

    def regress(self, x):
        raise LwbError("regress() on detached tensors is not part of the inference hot path; use forward()")


class ImpersonatorGenerator(NetworkBase):
    """Generator. Encoder-Decoder Architecture (networks/generator.py:187-320)."""

    def __init__(self, bg_dim, src_dim, tsf_dim, conv_dim=64, repeat_num=6):
        super(ImpersonatorGenerator, self).__init__()
        self._name = 'impersonator_generator'
        self.n_down = 3
        self.repeat_num = repeat_num
        self.bg_model = ResNetGenerator(conv_dim=conv_dim, c_dim=bg_dim, repeat_num=repeat_num, k_size=3, n_down=self.n_down)
        self.src_model = ResUnetGenerator(conv_dim=conv_dim, c_dim=src_dim, repeat_num=repeat_num, k_size=3, n_down=self.n_down)
        self.tsf_model = ResUnetGenerator(conv_dim=conv_dim, c_dim=tsf_dim, repeat_num=repeat_num, k_size=3, n_down=self.n_down)

    @torch.no_grad()
    def forward(self, bg_inputs, src_inputs, tsf_inputs, T):
        img_bg = self.bg_model(bg_inputs)
        src_img, src_mask, tsf_img, tsf_mask = self.infer_front(src_inputs, tsf_inputs, T)
        return img_bg, src_img, src_mask, tsf_img, tsf_mask

    def encode_src(self, src_inputs):
        _new_pass()
        return self.src_model.inference(src_inputs)

    @torch.no_grad()
    def infer_front(self, src_inputs, tsf_inputs, T):
        ac = K.default_align_corners()
        _new_pass()
        T = T.float().contiguous()
        src = self.src_model._stream(src_inputs, True, 'front')
        src.load_input(src_inputs.float())
        src.encode()
        src.resnets()
        tsf = self.tsf_model._stream(tsf_inputs, False, 'front')
        tsf.load_input(tsf_inputs.float())
        tsf.encode(warp_srcs=[None] + [a.f32 for a in src.e[1:]], T=T, ac=ac)
        tsf.resnets(warp_srcs=[a.f32 for a in src.res_out], T=T, ac=ac)
        src.decode()
        src_img, src_mask, _ = src.heads()
        tsf.decode()
        tsf_img, tsf_mask, _ = tsf.heads()
        return src_img, src_mask, tsf_img, tsf_mask

    @torch.no_grad()
    def swap(self, tsf_inputs, src_encoder_outs12, src_encoder_outs21, src_resnet_outs12, src_resnet_outs21, T12, T21, bg=None):
        """networks/generator.py:245-275.  With ``bg`` (extension) also returns the composite m*bg + (1-m)*color of
        models/swapper.py:268-269 from the head kernel."""
        ac = K.default_align_corners()
        _new_pass()
        T12, T21 = T12.float().contiguous(), T21.float().contiguous()
        tsf = self.tsf_model._stream(tsf_inputs, True, 'swap')
        tsf.load_input(tsf_inputs.float())
        enc = [None] + [((_nhwc_of(a), T12), (_nhwc_of(b), T21)) for a, b in zip(src_encoder_outs12[1:], src_encoder_outs21[1:])]
        res = [((_nhwc_of(a), T12), (_nhwc_of(b), T21)) for a, b in zip(src_resnet_outs12, src_resnet_outs21)]
        tsf.encode(warp_srcs=enc, ac=ac)
        tsf.resnets(warp_srcs=res, ac=ac)
        tsf.decode()
        tsf_img, tsf_mask, pred = tsf.heads(bg)
        if bg is not None:
            return tsf_img, tsf_mask, pred
        return tsf_img, tsf_mask

    @torch.no_grad()
    def inference(self, src_encoder_outs, src_resnet_outs, tsf_inputs, T, bg=None, pred_hwc=None, pred_u8=None):
        """networks/generator.py:277-301.  With ``bg`` also returns the composite of
        models/imitator.py:331 as a third value (fused into the head kernel); ``pred_hwc`` / ``pred_u8``
        (caller-allocated [B,H,W,3] float32 / uint8-BGR) receive the same frames in the layouts of the output
        path (models/imitator.py:178-180, utils/cv_utils.py:23-36) from that launch."""
        ac = K.default_align_corners()
        _new_pass()
        if (pred_hwc is not None or pred_u8 is not None) and bg is None:
            raise LwbError("pred_hwc / pred_u8 need bg (they hold the composite)")
        tsf_inputs = tsf_inputs.float().contiguous()
        T = T.float().contiguous()
        enc_w = [None] + [_nhwc_of(a) for a in src_encoder_outs[1:]]
        res_w = [_nhwc_of(a) for a in src_resnet_outs]
        B = tsf_inputs.shape[0]
        nsub = _sub_batches(B, enc_w, res_w, bg)

        def run(tag, x, Tx, outs):
            tsf = self.tsf_model._stream(x, False, tag)
            tsf.load_input(x)
            tsf.encode(warp_srcs=enc_w, T=Tx, ac=ac)
            tsf.resnets(warp_srcs=res_w, T=Tx, ac=ac)
            tsf.decode()
            return tsf.heads(bg, **outs)

        if nsub == 1:
            outs = {}
            if pred_hwc is not None or pred_u8 is not None:
                outs = dict(pred_hwc=pred_hwc, pred_u8=pred_u8)
            color, mask, pred = run('inference', tsf_inputs, T, outs)
        else:
            # LWB_STREAMS sub-batches on side streams: the HBM-bound kernels of one sub-batch (InstanceNorm / warp, heads
            # composite, input packing) co-run with the tensor-bound convolutions of the other, and the second wave of
            # the twelve 512-channel layers (128 tile pairs on 74 SM pairs) is filled by the other sub-batch's tiles.
            _, _, H, W = tsf_inputs.shape
            dev = tsf_inputs.device
            color = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev)
            mask = torch.empty((B, 1, H, W), dtype=torch.float32, device=dev)
            pred = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev) if bg is not None else None
            side = self.__dict__.setdefault('_lwb_side_streams', {})
            cur = torch.cuda.current_stream(dev)
            ready = torch.cuda.Event()
            ready.record(cur)
            step = B // nsub
            for i in range(nsub):
                if (dev, i) not in side:
                    side[(dev, i)] = torch.cuda.Stream(device=dev)
                st = side[(dev, i)]
                st.wait_event(ready)
                a, b = i * step, (i + 1) * step
                with torch.cuda.stream(st):
                    outs = dict(color=color[a:b], mask=mask[a:b])
                    if pred is not None:
                        outs['pred'] = pred[a:b]
                    if pred_hwc is not None:
                        outs['pred_hwc'] = pred_hwc[a:b]
                    if pred_u8 is not None:
                        outs['pred_u8'] = pred_u8[a:b]
                    run('inference#%d' % i, tsf_inputs[a:b], T[a:b], outs)
                    done = torch.cuda.Event()
                    done.record(st)
                cur.wait_event(done)
        if bg is not None:
            return color, mask, pred
        return color, mask

    def resize_trans(self, x, T):
        raise LwbError("resize_trans is fused into the warp kernels; call transform()/stn()")

    @torch.no_grad()
    def stn(self, x, T):
        return K.warp_nchw(x.float().contiguous(), T.float().contiguous(), align_corners=K.default_align_corners())

    @torch.no_grad()
    def transform(self, x, T):
        return K.warp_nchw(x.float().contiguous(), T.float().contiguous(), align_corners=K.default_align_corners())
