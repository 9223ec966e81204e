"""Seeded cases of the glue kernels around the conv engine, shared by test_glue_kernels_gpu.py (the CUDA front-ends of
impersonator_b200.kernels) and test_glue_cases_cpu.py (their torch stand-ins in kernel_emulator).

A case is one call of one front-end on CPU-built inputs.  ``run(api, put, alloc)`` makes the call through ``api`` (the
kernels module or the emulator); ``put`` moves an input to the device, ``alloc`` turns a CPU tensor into the caller buffer
the front-end writes (a sentinel-guarded view on the GPU).  The checks compare the outputs with a float64 restatement of
the operation from torch / numpy, never with the emulator:

* ``Bits``: exact contracts (layout moves, max, fp16 operand splits, uint8 truncation, range-flag bits);
* ``Tol``: |got - ref| <= tau * 2^-24 * S per element, S = the sum of |terms| (the same restatement on |inputs|) or, for
  elementwise operations, the magnitude the rounding scales with.  Each Tol also asserts tol < 0.1 * S / K for its K
  terms, so no bar is wide enough to hide a dropped, duplicated or shifted term.

Every required edge below names one case; the CPU suite checks that each front-end the emulator replaces has all its
edges, or an entry in COVERED_ELSEWHERE naming the test that covers it.
"""
import numpy as np
import torch
import torch.nn.functional as F

from conv_emulation import RANGE_VALUES, act_pair_blocks, fp16_pair

U32 = 2.0 ** -24               # fp32 unit roundoff
TAU = 16
NAN = float("nan")


# ------------------------------------------------------------------------------------------------------------ checks
def _get(outs, out):
    return out(outs) if callable(out) else outs[out]


class Tol(object):
    """``guard=False`` drops the tenth-of-one-term assertion for bars that grow with K (the attention sums), whose
    strength is shown by mutants instead.  A NaN reference wants NaN, an infinite one the same infinity.  ``ref`` and
    ``S`` may be functions, evaluated at the first check (the large references are not built at import); with
    ``of_outputs`` they are functions of the outputs, evaluated at every check (contracts stated on the kernel's own
    results, as Bits.want)."""

    def __init__(self, label, out, ref, S, K, tau=TAU, unit=U32, kernel_only=False, guard=True, of_outputs=False):
        self.label, self.out, self._ref, self._S, self.K = label, out, ref, S, K
        self.tau, self.unit, self.kernel_only, self.guard, self.of_outputs = tau, unit, kernel_only, guard, of_outputs

    @property
    def ref(self):
        if callable(self._ref):
            self._ref = self._ref()
        return self._ref.double()

    @property
    def S(self):
        if callable(self._S):
            self._S = self._S()
        return self._S.double()

    def ratio(self, case, outs):
        """-> the elementwise err / bar of the outputs (inf where a NaN or infinity is not matched)."""
        got = _get(outs, self.out).double()
        ref, S = (self._ref(outs).double(), self._S(outs).double()) if self.of_outputs else (self.ref, self.S)
        assert got.shape == ref.shape, "%s/%s: shape %s, want %s" % (case, self.label, tuple(got.shape), tuple(ref.shape))
        tol = self.tau * self.unit * S
        pos = (S > 0) & torch.isfinite(S)
        assert not self.guard or bool((tol[pos] < 0.1 * S[pos] / self.K).all()), \
            "%s/%s: tol %g * S is not below a tenth of one of the %d terms" % (case, self.label, self.tau * self.unit, self.K)
        err = (got - ref).abs()
        ratio = torch.where(tol > 0, err / tol.clamp(min=1e-300), torch.where(err > 0, float("inf"), 0.0))
        ratio = torch.where(torch.isnan(err) | torch.isnan(ratio), float("inf"), ratio)
        same = (got == ref) | (torch.isnan(got) & torch.isnan(ref))
        return torch.where(same, 0.0, ratio), err

    def __call__(self, case, outs):
        ratio, err = self.ratio(case, outs)
        err = torch.where(torch.isnan(err), 0.0, err)
        r = float(ratio.max()) if ratio.numel() else 0.0
        print("%s/%s: max err %.3g, max err/tol %.3f (K=%d)" % (case, self.label, float(err.max()) if err.numel() else 0.0, r, self.K))
        assert r <= 1.0, "%s/%s: error %.3g times the bar at %s" % (case, self.label, r, tuple(int(i) for i in np.unravel_index(
            int(ratio.flatten().argmax()), tuple(ratio.shape))))


class Bits(object):
    """Byte-identical to ``want`` (a tensor, or a function of the outputs for contracts stated on the kernel's own
    results)."""

    def __init__(self, label, out, want, kernel_only=False):
        self.label, self.out, self.want, self.kernel_only = label, out, want, kernel_only

    def __call__(self, case, outs):
        dense = lambda t: torch.empty(t.shape, dtype=t.dtype).copy_(t)           # noqa: E731 -- unit strides, size-1 dims too
        got = dense(_get(outs, self.out))
        want = dense(self.want(outs) if callable(self.want) else self.want)
        assert got.dtype == want.dtype and got.shape == want.shape, "%s/%s: %s %s, want %s %s" % (
            case, self.label, got.dtype, tuple(got.shape), want.dtype, tuple(want.shape))
        g, w = got.view(torch.uint8), want.view(torch.uint8)
        bad = (g != w).nonzero()
        print("%s/%s: %d of %d bytes differ" % (case, self.label, bad.shape[0], g.numel()))
        assert bad.shape[0] == 0, "%s/%s: first difference at byte %s (got %d, want %d)" % (
            case, self.label, tuple(bad[0].tolist()), int(g[tuple(bad[0])]), int(w[tuple(bad[0])]))


def Flag(want):
    return Bits("range_flag", "flag", torch.tensor([want], dtype=torch.int32))


class Case(object):
    def __init__(self, front, edge, run, checks, emulated=True):
        self.front, self.edge, self.run, self.checks, self.emulated = front, edge, run, checks, emulated
        self.name = "%s/%s" % (front, edge)


# ---------------------------------------------------------------------------------------------------------- helpers
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(g, *shape, scale=1.0, shift=0.0):
    return torch.randn(*shape, generator=g) * scale + shift


def _full(shape, value=NAN, dtype=torch.float32):
    return torch.full(shape, value, dtype=dtype)


def _put_all(put, *ts):
    return [put(t) if t is not None else None for t in ts]


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def u8_bgr(hwc):
    """cv_utils.save_cv2_img's ((img + 1) / 2.0 * 255).astype(np.uint8) in float32 numpy, channels reversed (RGB2BGR)."""
    a = hwc.numpy().astype(np.float32)
    return torch.from_numpy(((a + 1) / 2.0 * 255).astype(np.uint8)[..., ::-1].copy())


def _flow(g, n, th, tw):
    """Flow in [-1.1, 1.1] with about 15% of the pixels at -2 (the background code of the correspondence maps)."""
    T = torch.rand(n, th, tw, 2, generator=g) * 2.2 - 1.1
    bgm = torch.rand(n, th, tw, 1, generator=g) < 0.15
    return torch.where(bgm, torch.full_like(T, -2.0), T)


def _warp64(src_nchw, T, h, w, ac, n):
    """grid_sample(src, resize(T)) in float64 and its S: the bilinear terms on |src|, plus the tap weights' sensitivity
    to the fp32 rounding of the sample coordinate (about 2^-24 (h + w) pixels per tap, flow magnitudes up to 2)."""
    src = src_nchw.double().expand(n, -1, -1, -1)
    Ts = T.double()
    if tuple(Ts.shape[1:3]) != (h, w):
        Ts = _nhwc(F.interpolate(_nchw(Ts), size=(h, w), mode="bilinear", align_corners=True))
    val = F.grid_sample(src, Ts, mode="bilinear", padding_mode="zeros", align_corners=bool(ac))
    mag = F.grid_sample(src.abs(), Ts, mode="bilinear", padding_mode="zeros", align_corners=bool(ac))
    return val, mag + 8 * (h + w) * src.abs().amax(dim=(2, 3), keepdim=True)


# --------------------------------------------------------------------------------------------------------- norm_act
def _norm_act(edge, seed, n, h, w, c, mode="stats", relu=False, res_step=0, warp=None, post=None, lo_format=0, raw=None,
              flag=None):
    """mode: stats (InstanceNorm, gamma and beta) | affine (gamma, beta) | affine_g | affine_b | bare;
    warp: (src_batch, th, tw, align_corners); post: post_relu (bool) for the EXT variant's second affine."""
    g = _gen(seed)
    if raw is None:
        raw = _randn(g, n, h, w, c, scale=2.0, shift=0.5)
        if mode == "stats":                 # channel 0: mean 4e4 x its std (the fused x * scale + shift keeps ~1e-3)
            raw[..., 0] = _randn(g, n, h, w, shift=4e4)
    gamma = _randn(g, c, scale=0.1, shift=1.0) if mode in ("stats", "affine", "affine_g") else None
    beta = _randn(g, c, scale=0.1) if mode in ("stats", "affine", "affine_b") else None
    res = _randn(g, n, h * res_step, w * res_step, c) if res_step else None
    src = T = None
    if warp is not None:
        sb, th, tw, ac = warp
        src = _randn(g, sb, h, w, c)
        T = _flow(g, n, th, tw)
    ps = pt = None
    if post is not None:
        ps, pt = _randn(g, c, scale=0.2, shift=1.0), _randn(g, c, scale=0.3)

    x = raw.double()
    stats = None
    if mode == "stats":
        stats = torch.stack([x.sum(dim=(1, 2)), (x * x).sum(dim=(1, 2))], dim=-1)          # the conv epilogue's f64 sums
        mean = x.mean(dim=(1, 2))
        var = ((x - mean[:, None, None, :]) ** 2).mean(dim=(1, 2))
        scale = gamma.double() / torch.sqrt(var + 1e-5)
        shift = beta.double() - mean * scale
        sc, sh = scale[:, None, None, :], shift[:, None, None, :]
        y = x * sc + sh
        S = (x * sc).abs() + (mean[:, None, None, :] * sc).abs() + beta.double().abs()
    elif mode == "bare":
        y, S = x.clone(), x.abs()
    else:
        gm = gamma.double() if gamma is not None else 1.0
        bt = beta.double() if beta is not None else torch.zeros(c, dtype=torch.float64)
        y, S = x * gm + bt, (x * gm).abs() + bt.abs()
    K = 2
    if relu:
        y = y.clamp(min=0)
    if res is not None:
        r = res[:, ::res_step, ::res_step, :].double()
        y, S, K = y + r, S + r.abs(), K + 1
    if warp is not None:
        wv, ws_ = _warp64(_nchw(src), T, h, w, warp[3], n)
        y, S, K = y + _nhwc(wv), S + _nhwc(ws_), K + 4
    norm = mode != "bare"

    def run(api, put, alloc):
        o = {"y_f32": alloc(_full((n, h, w, c)))}
        o["hi"] = alloc(_full((n, h, w, c), dtype=torch.float16))
        o["lo"] = alloc(_full((n, h, w, c), dtype=torch.float16))
        if flag is not None:
            o["flag"] = alloc(torch.zeros(1, dtype=torch.int32))
        ws = alloc(torch.zeros(n, c, 2)) if norm else None
        r_, st, ga, be, re, sr, Td, psd, ptd = _put_all(put, raw, stats, gamma, beta, res, src, T, ps, pt)
        api.norm_act_nhwc(r_, st, ga, be, relu, ws, residual=re, warp_src=sr, T=Td,
                          align_corners=bool(warp[3]) if warp else False, y_f32=o["y_f32"], y_hi=o["hi"], y_lo=o["lo"],
                          lo_format=lo_format, post_scale=psd, post_shift=ptd, post_relu=bool(post),
                          res_step=res_step or 1, range_flag=o.get("flag"))
        return o

    if flag is not None:                 # the range cases: y = raw, only the flag bits matter (hi of NaN is not pinned)
        return Case("norm_act_nhwc", edge, run, [Bits("y_f32", "y_f32", raw), Flag(flag)])
    checks = [Bits("y_f32", "y_f32", raw) if (mode == "bare" and warp is None) else Tol("y_f32", "y_f32", y, S, K)]
    if post is None:
        checks.append(Bits("hi", "hi", lambda o: fp16_pair(o["y_f32"])[0]))
        if lo_format == 0:
            checks.append(Bits("lo", "lo", lambda o: fp16_pair(o["y_f32"])[1]))
        else:
            checks.append(Bits("lo8", lambda o: o["lo"].view(torch.uint8), lambda o: act_pair_blocks(o["y_f32"])))
    else:
        z = y * ps.double() + pt.double()
        if post:
            z = z.clamp(min=0)
        checks.append(Tol("hi+lo (post affine)", lambda o: o["hi"].double() + o["lo"].double(), z,
                          S * ps.double().abs() + pt.double().abs(), K + 1))
    return Case("norm_act_nhwc", edge, run, checks)


def norm_act_cases():
    cases = []
    for c in (8, 16, 64, 128, 256, 512, 1024, 2048):            # groups 1 .. 256; 105 pixels: a partial last block
        cases.append(_norm_act("stats c=%d" % c, 200 + c, 3, 7, 5, c, relu=True))
    cases += [
        _norm_act("affine gamma+beta", 301, 2, 5, 3, 64, mode="affine"),
        _norm_act("affine gamma only", 302, 2, 5, 3, 64, mode="affine_g", relu=True),
        _norm_act("affine beta only", 303, 2, 5, 3, 64, mode="affine_b"),                 # hmr.py: gamma=None, beta=bias
        _norm_act("bare", 304, 2, 3, 7, 128, mode="bare"),
        _norm_act("stats relu residual", 305, 2, 9, 4, 64, relu=True, res_step=1),
        _norm_act("bare warp", 306, 2, 6, 10, 32, mode="bare", warp=(1, 16, 20, 1)),      # generator.py _add_warp
        _norm_act("EXT post affine res_step 2", 307, 2, 5, 3, 64, mode="affine_b", res_step=2, post=True),
        _norm_act("EXT res_step 2", 308, 2, 5, 3, 64, relu=True, res_step=2),
        _norm_act("lo_format 1 c=512", 309, 1, 3, 5, 512, relu=True, lo_format=1),
    ]
    for sb in ("1", "n"):
        for tsize in ("same", "larger"):
            for ac in (0, 1):
                n, h, w = 2, 6, 10
                th, tw = (h, w) if tsize == "same" else (16, 20)
                cases.append(_norm_act("warp sb=%s T %s ac=%d" % (sb, tsize, ac), 310 + 4 * (sb == "n") + 2 * (tsize == "same") + ac,
                                       n, h, w, 32, relu=ac == 0, res_step=1 if sb == "n" else 0,
                                       warp=(1 if sb == "1" else n, th, tw, ac)))
    for label, v, want in RANGE_VALUES:
        raw = torch.rand(1, 3, 5, 8, generator=_gen(400)) * 8 - 4
        raw[0, 1, 2, 5] = v
        cases.append(_norm_act("range %s" % label, 400, 1, 3, 5, 8, mode="bare", raw=raw, flag=want))
    return cases


# --------------------------------------------------------------------------------------------------- instance_stats
def _instance_stats(edge, seed, n, h, w, c):
    x = _randn(_gen(seed), n, h, w, c, scale=3.0, shift=1.0)
    xd = x.double()
    ref = torch.stack([xd.sum(dim=(1, 2)), (xd * xd).sum(dim=(1, 2))], dim=-1)
    S = torch.stack([xd.abs().sum(dim=(1, 2)), (xd * xd).sum(dim=(1, 2))], dim=-1)

    def run(api, put, alloc):
        st = alloc(torch.zeros(n, c, 2, dtype=torch.float64))
        api.instance_stats_nhwc(put(x), st)
        return {"stats": st}
    # exact f64 sums of exact products: 8192 * 2^-53 ~ 1e-12 relative
    return Case("instance_stats_nhwc", edge, run, [Tol("stats", "stats", ref, S, h * w, tau=8192, unit=2.0 ** -53)],
                emulated=False)


def instance_stats_cases():
    return [_instance_stats("hw=35 c=40", 501, 2, 5, 7, 40),             # one split, hw % 8 != 0
            _instance_stats("hw=1000 c=96", 502, 2, 20, 50, 96),          # three splits
            _instance_stats("hw=16640 c=33", 503, 1, 128, 130, 33)]       # 64 splits, c % 32 != 0


# --------------------------------------------------------------------------------------------- heads / frames out
def _fold(raw, kw):
    """out[y, x, co] = sum_kx raw[y, x + kx - kw/2, kx*4 + co] over the columns inside the image."""
    if not kw:
        return raw[..., :4]
    w = raw.shape[2]
    r = torch.zeros(raw.shape[:3] + (4,), dtype=raw.dtype)
    for kx in range(kw):
        sh = kx - kw // 2
        x0, x1 = max(0, -sh), min(w, w - sh)
        if x1 > x0:
            r[:, :, x0:x1] += raw[:, :, x0 + sh:x1 + sh, kx * 4:kx * 4 + 4]
    return r


def sweep_values():
    """Float32 values at and a few ulps around every boundary 2k/255 - 1 of the uint8 cast, and +-1 exactly."""
    vals = [np.float32(-1.0), np.float32(1.0)]
    for k in range(256):
        b = np.float32(2.0 * k / 255.0 - 1.0)
        v = b
        for _ in range(4):
            v = np.nextafter(v, np.float32(-2))
            vals.append(v)
        vals.append(b)
        v = b
        for _ in range(4):
            v = np.nextafter(v, np.float32(2))
            vals.append(v)
    return torch.from_numpy(np.array(vals, dtype=np.float32))


def _sweep_frames(h, w):
    v = sweep_values()
    flat = torch.full((3 * h * w,), 0.5)
    flat[:v.numel()] = v
    return flat.view(1, 3, h, w)


def _heads(edge, seed, n, h, w, cs, kw, bg_batch, raw=None, bg=None, flag=0, flag_only=False):
    g = _gen(seed)
    if raw is None:
        raw = torch.rand(n, h, w, cs, generator=g) * 2 - 1           # folded sums stay below 7: range bit 2 clear
    if bg is None and not flag_only:
        bg = torch.rand(bg_batch, 3, h, w, generator=g) * 2 - 1

    def run(api, put, alloc):
        o = {"color": alloc(_full((n, 3, h, w))), "mask": alloc(_full((n, 1, h, w))), "flag": alloc(torch.zeros(1, dtype=torch.int32))}
        if bg is not None:
            o["pred"] = alloc(_full((n, 3, h, w)))
            o["pred_hwc"] = alloc(_full((n, h, w, 3)))
            o["pred_u8"] = alloc(torch.full((n, h, w, 3), 77, dtype=torch.uint8))
        api.heads_composite(put(raw), put(bg), color=o["color"], mask=o["mask"], pred=o.get("pred"), pred_hwc=o.get("pred_hwc"),
                            pred_u8=o.get("pred_u8"), folded_kw=kw, range_flag=o["flag"])
        return o

    if flag_only:
        return Case("heads_composite", edge, run, [Flag(flag)])
    r, Sr = _fold(raw.double(), kw), _fold(raw.double().abs(), kw)
    K = max(kw, 1)
    col, m = torch.tanh(_nchw(r[..., :3])), torch.sigmoid(_nchw(r[..., 3:]))
    Sc, Sm = _nchw(Sr[..., :3]), _nchw(Sr[..., 3:])
    b = bg.double().expand(n, -1, -1, -1)
    pred = m * b + (1 - m) * col
    checks = [Tol("color (tanh)", "color", col, Sc + col.abs(), K),
              Tol("mask (sigmoid)", "mask", m, Sm + m, K),
              Tol("pred", "pred", pred, (b.abs() + col.abs() + 1) * (Sc + Sm + 1), 2),
              Bits("pred_hwc", "pred_hwc", lambda o: _nhwc(o["pred"]).contiguous()),
              Bits("pred_u8", "pred_u8", lambda o: u8_bgr(o["pred_hwc"])),
              Flag(flag)]
    return Case("heads_composite", edge, run, checks)


def heads_cases():
    cases = []
    for w in (1, 2, 3, 70):                # w = 2: the folded columns reach past both borders of a pixel
        for kw, cs, bgb in ((0, 4, "1"), (0, 32, "n"), (7, 32, "1"), (7, 32, "n")):
            cases.append(_heads("kw=%d w=%d c_stride=%d bg_batch=%s" % (kw, w, cs, bgb), 600 + w + kw + cs, 2, 3, w, cs, kw,
                                1 if bgb == "1" else 2))
    # the composite is bg exactly where the mask saturates to 1 (|pre-activation| 20 also sets range bit 2)
    h, w = 13, 60
    raw = torch.rand(1, h, w, 4, generator=_gen(650)) * 2 - 1
    raw[..., 3] = 20.0
    cases.append(_heads("u8 sweep", 650, 1, h, w, 4, 0, 1, raw=raw, bg=_sweep_frames(h, w), flag=4))
    for label, v, ch, want in (("8.0", 8.0, 0, 4), ("below 8.0", float(np.nextafter(np.float32(8), np.float32(0))), 1, 0),
                               ("-8.0", -8.0, 3, 4), ("nan", NAN, 2, 4)):
        raw = torch.rand(1, 2, 3, 4, generator=_gen(660)) * 2 - 1
        raw[0, 1, 2, ch] = v
        cases.append(_heads("range %s" % label, 660, 1, 2, 3, 4, 0, 1, raw=raw, flag=want, flag_only=True))
    return cases


def frames_out_cases():
    frames = _sweep_frames(13, 60)

    def run(api, put, alloc):
        hwc, u8 = api.frames_out(put(frames), want_hwc=True, want_u8=True)
        return {"hwc": hwc, "u8": u8}
    return [Case("frames_out", "u8 sweep", run, [Bits("hwc", "hwc", _nhwc(frames).contiguous()),
                                                 Bits("u8", "u8", u8_bgr(_nhwc(frames)))], emulated=False)]


# ------------------------------------------------------------------------------------------------------ direct conv
def _conv_direct(edge, seed, n, cin, h, w, cout, k, stride=1, pad=0, dil=1, bias=True):
    g = _gen(seed)
    x, wt = _randn(g, n, cin, h, w), _randn(g, cout, cin, k, k, scale=0.2)
    b = _randn(g, cout) if bias else None
    conv = lambda a, ww, bb: F.conv2d(a, ww, bb, stride=stride, padding=pad, dilation=dil)      # noqa: E731
    ref = conv(x.double(), wt.double(), b.double() if bias else None)
    S = conv(x.double().abs(), wt.double().abs(), b.double().abs() if bias else None)

    def run(api, put, alloc):
        return {"out": api.conv2d_direct_nchw(put(x), put(wt), put(b) if bias else None, stride=stride, pad=pad, dil=dil)}
    return Case("conv2d_direct_nchw", edge, run, [Tol("out", "out", ref, S, cin * k * k + 1)])


def conv_direct_cases():
    return [_conv_direct("cout=7", 701, 2, 5, 9, 8, 7, 3, pad=1),
            _conv_direct("dilation 2", 702, 1, 5, 12, 10, 4, 3, pad=2, dil=2),
            _conv_direct("stride 2 odd sizes", 703, 2, 3, 9, 11, 5, 3, stride=2, pad=1),
            _conv_direct("pad > k/2", 704, 1, 4, 6, 7, 4, 3, pad=3),
            _conv_direct("bias None", 705, 2, 5, 8, 8, 6, 3, pad=1, bias=False),
            _conv_direct("1x1", 706, 2, 6, 7, 5, 9, 1),
            _conv_direct("inpaintor 5x5", 707, 1, 5, 20, 20, 8, 5, pad=2),
            _conv_direct("inpaintor 4x4 s2", 708, 1, 8, 20, 20, 6, 4, stride=2, pad=1),
            _conv_direct("inpaintor 3x3 dil 16", 709, 1, 6, 40, 36, 5, 3, pad=16, dil=16)]


# --------------------------------------------------------------------------------------------------------- 7x7 heads
def _heads7x7(edge, seed, n, h, w):
    g = _gen(seed)
    x = _randn(g, n, h, w, 64)
    wi, wa = _randn(g, 3, 64, 7, 7, scale=0.02), _randn(g, 1, 64, 7, 7, scale=0.02)
    wt = torch.cat([wi, wa]).double()
    ref = _nhwc(F.conv2d(_nchw(x.double()), wt, padding=3))
    S = _nhwc(F.conv2d(_nchw(x.double().abs()), wt.abs(), padding=3))

    def run(api, put, alloc):
        out = alloc(_full((n, h, w, 4)))
        api.conv7x7_heads_nhwc(put(x), api.pack_head_weights(put(wi), put(wa)), out=out)
        return {"out": out}
    return Case("conv7x7_heads_nhwc", edge, run, [Tol("out", "out", ref, S, 64 * 49)])


def heads7x7_cases():
    return [_heads7x7("1x1", 801, 2, 1, 1), _heads7x7("5x3", 802, 2, 5, 3), _heads7x7("17x65", 803, 1, 17, 65)]


# --------------------------------------------------------------------------------------------------------- gated BN
def _gated_bn(act, with_scale, seed):
    g = _gen(seed)
    n, c, h, w = 2, 5, 3, 7
    ab = _randn(g, n, 2 * c, h, w, scale=2.0)
    sc, sh = (_randn(g, c, scale=0.3, shift=1.0), _randn(g, c, scale=0.5)) if with_scale else (None, None)
    a, gt = ab[:, :c].double(), ab[:, c:].double()
    a = F.leaky_relu(a, 0.2) if act == 2 else (a.clamp(min=0) if act == 1 else a)
    y = a * torch.sigmoid(gt)
    S = y.abs()
    if with_scale:
        y = y * sc.double()[None, :, None, None] + sh.double()[None, :, None, None]
        S = S * sc.double().abs()[None, :, None, None] + sh.double().abs()[None, :, None, None]

    def run(api, put, alloc):
        return {"out": api.gated_bn_nchw(put(ab), act, put(sc) if with_scale else None, put(sh) if with_scale else None)}
    # sigmoid through expf and a division, the product, the fused affine: a few ulps of S
    return Case("gated_bn_nchw", "act=%d %s" % (act, "scale" if with_scale else "no scale"), run,
                [Tol("out", "out", y, S, 2 if with_scale else 1)])


def gated_bn_cases():
    return [_gated_bn(act, s, 900 + 2 * act + s) for act in (0, 1, 2) for s in (False, True)]


# ---------------------------------------------------------------------------------------------------- max pool (HMR)
def _maxpool(edge, seed, n, c, h, w, k, s):
    x = _randn(_gen(seed), n, c, h, w)
    ref = _nhwc(F.max_pool2d(x, kernel_size=k, stride=s, ceil_mode=True)).contiguous()

    def run(api, put, alloc):
        out = alloc(_full(tuple(ref.shape)))
        api.maxpool_nchw_to_nhwc(put(x), k, s, out=out)
        return {"out": out, "allocated": api.maxpool_nchw_to_nhwc(put(x), k, s)}
    return Case("maxpool_nchw_to_nhwc", edge, run, [Bits("out", "out", ref), Bits("allocated", "allocated", ref)])


def maxpool_cases():
    return [_maxpool("112 -> 56 clipped last window", 1001, 1, 3, 112, 112, 3, 2),
            _maxpool("h = k", 1002, 2, 4, 3, 5, 3, 2),
            _maxpool("k < stride", 1003, 2, 3, 4, 5, 1, 2)]                      # torch: 2 x 3 windows, not 3 x 3


# ---------------------------------------------------------------------------------------------- global average pool
def _avgpool(edge, seed, n, h, w, c, ld, scale, relu):
    g = _gen(seed)
    x = _randn(g, n, h, w, c, scale=2.0)
    sc, sh = (_randn(g, c, scale=0.3, shift=1.0), _randn(g, c, scale=0.5)) if scale else (None, None)
    v = x.double() * sc.double() + sh.double() if scale else x.double()
    Sv = (x.double() * sc.double()).abs() + sh.double().abs() if scale else x.double().abs()
    if relu:
        v = v.clamp(min=0)
    init = _full((n, ld))

    def run(api, put, alloc):
        buf = alloc(init)
        api.global_avgpool_nhwc(put(x), put(sc) if scale else None, put(sh) if scale else None, relu=relu, out=buf, ld_out=ld)
        return {"out": buf[:, :c], "pad": buf[:, c:]}
    return Case("global_avgpool_nhwc", edge, run, [Tol("out", "out", v.mean(dim=(1, 2)), Sv.mean(dim=(1, 2)), 2 * h * w + 1),
                                                   Bits("columns >= c untouched", "pad", init[:, c:])])


def avgpool_cases():
    return [_avgpool("scale relu ld_out > c", 1101, 2, 7, 7, 40, 48, True, True),
            _avgpool("no scale hw=1", 1102, 3, 1, 1, 20, 20, False, False),
            _avgpool("scale no relu", 1103, 1, 5, 9, 70, 70, True, False)]


# ----------------------------------------------------------------------------------------------------------- linear
def _linear(edge, seed, n, k, m, ld_x=None, ld_out=None, bias=True, relu=False, acc=False):
    g = _gen(seed)
    ld_x, ld_out = ld_x or k, ld_out or m
    xfull = _randn(g, n, ld_x)
    wt = _randn(g, m, k, scale=k ** -0.5)
    b = _randn(g, m) if bias else None
    init = _randn(g, n, ld_out) if acc else _full((n, ld_out))
    x = xfull[:, :k].double()
    y = x @ wt.double().t() + (b.double() if bias else 0.0)
    S = x.abs() @ wt.double().abs().t() + (b.double().abs() if bias else 0.0)
    if relu:
        y = y.clamp(min=0)
    if acc:
        y, S = y + init[:, :m].double(), S + init[:, :m].double().abs()

    def run(api, put, alloc):
        buf = alloc(init)
        api.linear(put(xfull)[:, :k], put(wt), put(b) if bias else None, relu=relu, out=buf[:, :m], accumulate=acc)
        return {"out": buf[:, :m], "pad": buf[:, m:]}
    return Case("linear", edge, run, [Tol("out", "out", y, S, k + 2), Bits("columns >= m untouched", "pad", init[:, m:])])


def linear_cases():
    return [_linear("k=1", 1201, 3, 1, 5, relu=True),
            _linear("k=31 ld_x > k bias None", 1202, 2, 31, 7, ld_x=40, bias=False),
            _linear("k=85 m=1 ld_out > m", 1203, 4, 85, 1, ld_out=3, relu=True),
            _linear("k=2133", 1204, 2, 2133, 9, relu=True),
            # HMR's third regressor layer: theta += fc3(h2), theta a column slice of [features | theta]
            _linear("accumulate into a slice", 1205, 2, 1024, 85, ld_out=2133, acc=True)]


# ----------------------------------------------------------------------------------------------------------- LPIPS
_LPIPS_SHIFT, _LPIPS_SCALE = (-.030, -.088, -.188), (.458, .448, .450)


def _lpips_input(from01, seed):
    g = _gen(seed)
    n, h, w = 2, 5, 7
    lo = 0.0 if from01 else -1.0
    pred = torch.rand(n, 3, h, w, generator=g) * (1 - lo) + lo
    ref = torch.rand(n, 3, h, w, generator=g) * (1 - lo) + lo
    pred[0, :, 0, :2], ref[1, :, 4, 6] = lo, 1.0                   # the ends of the range
    x = torch.cat([pred, ref])
    if from01:
        x = x * 2 - 1
    want = (x - torch.tensor(_LPIPS_SHIFT).view(1, 3, 1, 1)) / torch.tensor(_LPIPS_SCALE).view(1, 3, 1, 1)

    def run(api, put, alloc):
        out = alloc(_full((2 * n, 3, h, w)))
        api.lpips_input(put(pred), put(ref), from01=from01, out=out)
        return {"out": out}
    return Case("lpips_input", "from01=%d" % from01, run, [Bits("out", "out", want)])


def _lpips_layer(edge, seed, n, h, w, c, layer, L=3):
    g = _gen(seed)
    feat = _randn(g, 2 * n, h, w, c).clamp(min=0) * 3                 # post-ReLU features
    if h * w > 1:
        feat[n + 1, 0, 1] = 0.0                                        # one ref pixel all zero, its pred pixel not
    lin = torch.rand(c, generator=g) * 0.2
    layers0 = _randn(g, n, L)
    score0 = _randn(g, n).abs()
    f = feat.double()
    fn = f / (f.pow(2).sum(-1, keepdim=True).sqrt() + 1e-10)
    d = fn[n:] - fn[:n]
    v = (d * d * lin.double()).sum(-1).mean(dim=(1, 2))
    Sv = ((fn[n:].abs() + fn[:n].abs()) ** 2 * lin.double()).sum(-1).mean(dim=(1, 2))
    score = v + score0.double() if layer > 0 else v
    Ss = Sv + score0.double().abs() if layer > 0 else Sv
    others = [k for k in range(L) if k != layer]

    def run(api, put, alloc):
        layers, sc = alloc(layers0), alloc(score0)
        api.lpips_layer(put(feat), put(lin), layer, layers, sc)
        return {"layer": layers[:, layer], "others": layers[:, others], "score": sc}
    return Case("lpips_layer", edge, run, [Tol("layers[:, %d]" % layer, "layer", v, Sv, c * h * w),
                                           Bits("other layers untouched", "others", layers0[:, others]),
                                           Tol("score", "score", score, Ss, c * h * w + 1)])


def lpips_cases():
    return [_lpips_input(False, 1301), _lpips_input(True, 1302),
            _lpips_layer("c=40 zero pixel layer 0", 1303, 2, 5, 7, 40, 0),
            _lpips_layer("hw=1 layer 2 accumulates", 1304, 3, 1, 1, 40, 2)]


# ------------------------------------------------------------------------------------------------- layout / warp
def _nhwc_to_nchw(edge, seed, n, h, w, c, cs):
    x = _randn(_gen(seed), n, h, w, cs)

    def run(api, put, alloc):
        out = alloc(_full((n, c, h, w)))
        api.nhwc_to_nchw(put(x), c=c, out=out)
        return {"out": out}
    return Case("nhwc_to_nchw", edge, run, [Bits("out", "out", _nchw(x[..., :c]).contiguous())])


def _warp_nchw(edge, seed, sb, B, C, h, w, th, tw, ac, acc):
    g = _gen(seed)
    x = _randn(g, sb, C, h, w)
    T = _flow(g, B, th, tw)
    init = _randn(g, B, C, h, w) if acc else _full((B, C, h, w))
    ref, S = _warp64(x, T, h, w, ac, B)
    if acc:
        ref, S = ref + init.double(), S + init.double().abs()

    def run(api, put, alloc):
        out = alloc(init)
        api.warp_nchw(put(x), put(T), align_corners=bool(ac), out=out, accumulate=acc)
        return {"out": out}
    return Case("warp_nchw", edge, run, [Tol("out", "out", ref, S, 5 if acc else 4)])


def layout_warp_cases():
    return [_nhwc_to_nchw("c=4 c_stride=32", 1401, 2, 3, 5, 4, 32),
            _nhwc_to_nchw("c=100 hw=37x3", 1402, 2, 37, 3, 100, 104),
            _warp_nchw("accumulate src_batch=B C=70", 1403, 2, 2, 70, 9, 13, 16, 16, 1, True),
            _warp_nchw("src_batch=1 T same size", 1404, 1, 3, 5, 12, 7, 12, 7, 0, False)]


# ------------------------------------------------------------------------------------------------ self attention
ATT_DQ, ATT_DV = 16, 128
ATT_SIZES = {1: (1, 1), 63: (7, 9), 64: (8, 8), 65: (5, 13), 129: (3, 43), 4096: (64, 64)}


def attention64(qkv, bias, x, gamma, dq=ATT_DQ):
    """gamma * softmax(q k^T) v + x in float64, and its S: the same sums on |v| and |x| with the softmax weights
    unchanged.  -> (ref, S) as [n, h, w, dv]."""
    n, h, w, _ = qkv.shape
    dv = x.shape[3]
    t = (qkv[..., :2 * dq + dv].double() + bias.double()).view(n, h * w, -1)
    q, k, v = t[..., :dq], t[..., dq:2 * dq], t[..., 2 * dq:]
    p = torch.softmax(torch.bmm(q, k.transpose(1, 2)), dim=-1)
    g, xd = gamma.double(), x.double().view(n, h * w, dv)
    ref = g * torch.bmm(p, v) + xd
    S = g.abs() * torch.bmm(p, v.abs()) + xd.abs()
    return ref.view(n, h, w, dv), S.view(n, h, w, dv)


def _attention(edge, seed, n, N, qk="rand", ld=ATT_DQ * 2 + ATT_DV, gamma=0.7, zero_x=False, nan_pad=False):
    """qk: rand (logits about +-5) | uniform (q = 0) | big_first / big_last (one key 30 above the rest, in the first tile
    or in the last, partial one) | ascending (every key's logit above the last, for every query) | span80 (logits
    spread over +-80: most exp terms underflow) | ties (four distinct keys, each repeated)."""
    g = _gen(seed)
    h, w = ATT_SIZES[N]
    qkv = _randn(g, n, h, w, ld)
    bias = _randn(g, ATT_DQ * 2 + ATT_DV, scale=0.1)
    x = torch.zeros(n, h, w, ATT_DV) if zero_x else _randn(g, n, h, w, ATT_DV)
    q, k = qkv[..., :ATT_DQ], qkv[..., ATT_DQ:2 * ATT_DQ]              # views: edits land in qkv
    if qk == "rand":
        q.mul_(0.6)
    elif qk == "uniform":
        q.copy_(-bias[:ATT_DQ].expand_as(q))                             # q + bias_q = 0 exactly: every logit is 0
    else:
        # every query a positive multiple of one direction u: a key's logit order is the same for all queries
        u = _randn(g, ATT_DQ)
        u = u / u.norm()
        q.copy_(u * (0.5 + torch.rand(n, h, w, 1, generator=g)) - bias[:ATT_DQ])
        t = torch.randn(n, N, generator=g)
        if qk in ("big_first", "big_last"):
            t[:, 0 if qk == "big_first" else N - 1] = 30.0
        elif qk == "ascending":
            t = torch.linspace(-4, 4, N).expand(n, N).clone()
        elif qk == "span80":
            t = torch.linspace(-80, 80, N)[torch.randperm(N, generator=g)].expand(n, N).clone()
        elif qk == "ties":
            t = torch.tensor([1.5, -0.5, 1.5, 0.25])[torch.arange(N) % 4].expand(n, N).clone()
        kk = t[..., None] * u + 0.05 * _randn(g, n, N, ATT_DQ) * (qk not in ("ties", "ascending"))
        k.copy_(kk.view(n, h, w, ATT_DQ) - bias[ATT_DQ:2 * ATT_DQ])
    if nan_pad:
        qkv[..., 2 * ATT_DQ + ATT_DV:] = NAN
    gm = torch.tensor([gamma])
    ref_S = []

    def ref(i):                                          # built at the first check, not at import
        if not ref_S:
            ref_S.extend(attention64(qkv, bias, x, gm))
        return ref_S[i]

    def run(api, put, alloc):
        out = alloc(_full((n, h, w, ATT_DV)))
        api.self_attention_nhwc(put(qkv), put(bias), put(x), put(gm), out=out)
        return {"out": out}
    if gamma == 0:
        return Case("self_attention_nhwc", edge, run, [Bits("out == x", "out", x)])
    # The kernel sums the N keys one after the other in fp32: the weights l and each accumulator channel are sequential
    # sums of N terms, every term rescaled by a running product of up to N factors exp(m_old - m_new).  The deterministic
    # bound of such a sum is about N u S (Higham's gamma_N); tau = 16 covers the logit's own 16-term dot, the exp
    # evaluations and the final fmaf.  At N = 4096 the bar is no longer below one term (the tenth-of-a-term guard cannot
    # hold), so test_attention_mutants_cpu.py shows on these cases that a dropped tile, a missed rescale or a mixed-up
    # value slot each exceed it.
    return Case("self_attention_nhwc", edge, run, [Tol("out", "out", lambda: ref(0), lambda: ref(1), N, tau=TAU * N,
                                                                    guard=False)])


def attention_cases():
    cases = [_attention("N=%d" % N, 1500 + N % 100, 2, N) for N in (1, 63, 64, 65, 129, 4096)]
    cases += [
        _attention("N=65 n=3", 1510, 3, 65),
        _attention("uniform logits", 1511, 2, 129, qk="uniform"),
        _attention("big key in the first tile", 1512, 2, 129, qk="big_first"),
        _attention("big key in the last partial tile", 1513, 2, 129, qk="big_last"),
        _attention("ascending logits", 1514, 2, 129, qk="ascending"),
        _attention("logits span +-80", 1515, 2, 129, qk="span80"),
        _attention("exact ties", 1516, 2, 129, qk="ties"),
        _attention("gamma=0", 1517, 2, 65, gamma=0.0),
        _attention("gamma<0", 1518, 2, 65, gamma=-1.3),
        _attention("x=0", 1519, 2, 65, zero_x=True),
        _attention("ld=176 NaN pad", 1520, 2, 65, ld=176, nan_pad=True),
    ]
    return cases


ATTENTION_EDGES = ["N=%d" % N for N in (1, 63, 64, 65, 129, 4096)] + [
    "N=65 n=3", "uniform logits", "big key in the first tile", "big key in the last partial tile", "ascending logits",
    "logits span +-80", "exact ties", "gamma=0", "gamma<0", "x=0", "ld=176 NaN pad"]


# -------------------------------------------------------------------------------------------------- gated epilogue
def _pin_nan(got, want):
    """``want`` with its NaN entries replaced by ``got``'s where that is NaN too: any NaN payload is the same NaN."""
    both = torch.isnan(want.float()) & torch.isnan(got.float())
    return torch.where(both, got, want)


def _up2(t, up):
    return t.repeat_interleave(up, dim=1).repeat_interleave(up, dim=2) if up == 2 else t


def _gated(edge, seed, n, h, w, c, cs, up=1, outputs="f32 hi lo", lo_format=0, bias=True, act=2, scale=True, clamp=False,
           f32_extra=0, c_pad=None, raw=None, gates=None, flag=None, wide=1.0):
    """outputs: the buffers passed (f32 and / or operands hi [+ lo]); f32_extra: columns of the f32 buffer past c, which
    must keep their sentinel; gates: values written over the first gate channels; flag: the range_flag bits wanted."""
    g = _gen(seed)
    outs_on = outputs.split()
    c_pad = c_pad or ((c + 63) // 64 * 64)
    if raw is None:
        raw = _randn(g, n, h, w, cs, scale=2.0 * wide)
    if gates is not None:
        flat = raw[..., c:2 * c].reshape(-1)
        flat[:len(gates)] = torch.tensor(gates)
        raw[..., c:2 * c] = flat.view(n, h, w, c)
    b = _randn(g, 2 * c, scale=0.3) if bias else None
    sc, sh = (_randn(g, c, scale=0.3, shift=1.0), _randn(g, c, scale=0.2)) if scale else (None, None)

    rd = raw.double()
    a, gt = rd[..., :c], rd[..., c:2 * c]
    Sa, Sg = a.abs(), gt.abs()
    if bias:
        a, gt = a + b.double()[:c], gt + b.double()[c:]
        Sa, Sg = Sa + b.double()[:c].abs(), Sg + b.double()[c:].abs()
    if act == 2:
        Sa = torch.where(a < 0, 0.2 * Sa, Sa)
        a = F.leaky_relu(a, 0.2)
    sig = torch.sigmoid(gt)
    # d sigmoid = sigmoid (1 - sigmoid) d gate; expf(-gate) overflows below a gate of -88.7, where the kernel's 0 is
    # within 2^-127 of the sigmoid: 2^-100 * tau * u covers that
    dsig = torch.where(sig * (1 - sig) > 0, sig * (1 - sig) * Sg, torch.zeros_like(sig))
    y, S = a * sig, Sa * (sig + dsig + 2.0 ** -100)
    if scale:
        y, S = y * sc.double() + sh.double(), S * sc.double().abs() + sh.double().abs()
    if clamp:
        y = y.clamp(-1, 1)
    y, S = _up2(y, up), _up2(S, up)
    ho, wo = h * up, w * up
    init_f32 = _full((n, ho, wo, c + f32_extra))

    def call(api, put, alloc, o, f32, hi, lo):
        api.gated_act_nhwc(put(raw), c, put(b), act, put(sc), put(sh), upsample=up, clamp=clamp, y_f32=f32, y_hi=hi, y_lo=lo,
                           lo_format=lo_format, range_flag=o.get("flag"))

    def run(api, put, alloc):
        o = {}
        if flag is not None:
            o["flag"] = alloc(torch.zeros(1, dtype=torch.int32))
        if "f32" in outs_on:
            o["f32"] = alloc(init_f32)
        if "hi" in outs_on:
            o["hi"] = alloc(_full((n, ho, wo, c_pad), dtype=torch.float16))
            if "lo" in outs_on:
                o["lo"] = alloc(_full((n, ho, wo, c_pad), dtype=torch.float16))
        call(api, put, alloc, o, o.get("f32"), o.get("hi"), o.get("lo"))
        if "f32" not in outs_on:              # the same call with an f32 output: the value the operands must split
            o["f32"] = alloc(init_f32)
            call(api, put, alloc, {}, o["f32"], None, None)
        return o

    checks = [Tol("y_f32", lambda o: o["f32"][..., :c], y, S, 3)]
    if f32_extra:
        checks.append(Bits("f32 columns >= c untouched", lambda o: o["f32"][..., c:], init_f32[..., c:]))
    if flag is not None:
        checks.append(Flag(flag))
    if "hi" in outs_on:
        def v_pad(o):
            v = torch.zeros(n, ho, wo, c_pad)
            v[..., :c] = o["f32"][..., :c]
            return v
        checks.append(Bits("hi", "hi", lambda o: _pin_nan(o["hi"], fp16_pair(v_pad(o))[0])))
        if "lo" in outs_on and lo_format == 0:
            checks.append(Bits("lo", "lo", lambda o: _pin_nan(o["lo"], fp16_pair(v_pad(o))[1])))
        elif "lo" in outs_on:
            checks.append(Bits("lo8", lambda o: o["lo"].view(torch.uint8), lambda o: act_pair_blocks(v_pad(o))))
    return Case("gated_act_nhwc", edge, run, checks)


def inpaintor_gated_bindings():
    """Every (c, c_stride, up, outputs, lo_format) the inpaintor binds at 256x256 in the three precision modes, from
    _InpaintStream over InpaintSANet's module tree.  CPU only: needs kernel_emulator's stand-ins installed."""
    from impersonator_b200.inpaintor import InpaintSANet, _InpaintStream
    net = InpaintSANet(c_dim=4).eval()
    combos = set()
    for split in (0, 1, 2):
        st = _InpaintStream(net, 1, 256, 256, torch.device("cpu"), split)
        for r in st.coarse + st.refine + st.upsample:
            outs = ["f32"] if r["y_f32"] is not None else []
            if r["out"] is not None:
                outs += ["hi"] + (["lo"] if r["out"].lo is not None else [])
            combos.add((r["c"], r["conv"].out.shape[3], r["up"], " ".join(outs), st.lo_format))
    return sorted(combos)


# (c, c_stride, up, outputs, lo_format) of inpaintor_gated_bindings(); test_glue_cases_cpu.py checks the list is complete
INPAINTOR_GATED = [
    (3, 16, 1, "f32", 0), (3, 16, 1, "f32", 1),
    (16, 32, 1, "hi", 0), (16, 32, 1, "hi lo", 0), (16, 32, 1, "hi lo", 1),
    (32, 64, 1, "hi", 0), (32, 64, 1, "hi lo", 0), (32, 64, 1, "hi lo", 1),
    (64, 128, 1, "hi", 0), (64, 128, 1, "hi lo", 0), (64, 128, 1, "hi lo", 1),
    (64, 128, 2, "hi", 0), (64, 128, 2, "hi lo", 0), (64, 128, 2, "hi lo", 1),
    (128, 256, 1, "hi", 0), (128, 256, 1, "hi lo", 0), (128, 256, 1, "hi lo", 1),
    (128, 256, 1, "f32 hi", 0), (128, 256, 1, "f32 hi lo", 0), (128, 256, 1, "f32 hi lo", 1),
    (128, 256, 2, "hi", 0), (128, 256, 2, "hi lo", 0), (128, 256, 2, "hi lo", 1),
]


def _binding_edge(cb):
    return "inpaintor c=%d c_stride=%d up=%d %s lo_format=%d" % cb


def _gated_range(edge, v, want, outputs="f32 hi lo"):
    """act none, no bias / scale, gate +inf (sigmoid exactly 1): y = a exactly, one channel of one pixel at v."""
    raw = torch.rand(1, 3, 5, 16, generator=_gen(1600)) * 8 - 4
    raw[..., 8:] = float("inf")
    raw[0, 1, 2, 5] = v
    return _gated(edge, 1600, 1, 3, 5, 8, 16, outputs=outputs, bias=False, act=0, scale=False, raw=raw, flag=want)


def gated_cases():
    cases = [_gated(_binding_edge(cb), 1700 + i, 2, 5, 7, cb[0], cb[1], up=cb[2], outputs=cb[3], lo_format=cb[4],
                    scale=cb[0] != 3, act=0 if cb[0] == 3 else 2, clamp=cb[0] == 3, wide=2.0 if cb[0] == 3 else 1.0)
             for i, cb in enumerate(INPAINTOR_GATED)]
    cases += [
        _gated("c=3 f32 only", 1801, 2, 4, 6, 3, 8, outputs="f32"),
        _gated("c=16 f32 only f32_stride=21", 1802, 2, 4, 6, 16, 40, outputs="f32", f32_extra=5),
        _gated("c=3 f32_stride=8", 1803, 1, 3, 5, 3, 6, outputs="f32", f32_extra=5),
        _gated("up=2 odd h w lo_format=0", 1804, 2, 5, 7, 24, 48, up=2, lo_format=0),
        _gated("up=2 odd h w lo_format=1", 1805, 2, 5, 7, 24, 48, up=2, lo_format=1),
        _gated("no bias", 1806, 2, 3, 5, 16, 32, bias=False),
        _gated("no scale", 1807, 2, 3, 5, 16, 32, scale=False),
        _gated("act none", 1808, 2, 3, 5, 16, 32, act=0),
        _gated("clamp beyond +-1", 1809, 2, 3, 5, 16, 32, clamp=True, wide=3.0),
        _gated("bare", 1810, 2, 3, 5, 16, 32, bias=False, scale=False, act=0),
        _gated("gates +-100 +-inf nan", 1811, 1, 3, 5, 16, 32, clamp=True, flag=3,
               gates=[100.0, -100.0, float("inf"), float("-inf"), NAN, 89.0, -89.0, -88.0]),
    ]
    cases += [_gated_range("range %s" % label, v, want) for label, v, want in RANGE_VALUES]
    cases.append(_gated_range("range 65520 no operand output", 65520.0, 0, outputs="f32"))
    return cases


GATED_EDGES = [_binding_edge(cb) for cb in INPAINTOR_GATED] + [
    "c=3 f32 only", "c=16 f32 only f32_stride=21", "c=3 f32_stride=8", "up=2 odd h w lo_format=0", "up=2 odd h w lo_format=1",
    "no bias", "no scale", "act none", "clamp beyond +-1", "bare", "gates +-100 +-inf nan"] + [
    "range %s" % label for label, _, _ in RANGE_VALUES] + ["range 65520 no operand output"]


# ------------------------------------------------------------------------------------------------------------- SMPL
SMPL_PARENTS = [-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21]    # depth 9 (0..22)
SMPL_NJ, SMPL_NPF, SMPL_NREG = 24, 207, 19
SMPL_TAU = 2


def smpl_model(seed, V, nb=10, sparse=False, blend=4.0):
    """A seeded random SMPL model in the oracle's layout (float32 values): 24 joints, 207 pose bases; dense skin
    weights, or two joints per vertex when sparse.  blend scales the blend shapes above the synthetic model's
    (|shapedirs| ~ 0.03, |posedirs| ~ 0.017), so that dropping one beta or a quarter of the pose terms moves the vertices
    by more than 10 bars (test_smpl_cases_cpu.py)."""
    g = _gen(seed)
    w = torch.rand(V, SMPL_NJ, generator=g) ** 4
    if sparse:
        keep = torch.zeros(V, SMPL_NJ, dtype=torch.bool)
        for _ in range(2):
            keep[torch.arange(V), torch.randint(SMPL_NJ, (V,), generator=g)] = True
        w = torch.where(keep, w + 0.1, torch.zeros_like(w))
    jr = torch.rand(V, SMPL_NJ, generator=g)
    reg = torch.zeros(V, SMPL_NREG)
    for j in range(SMPL_NREG):                                   # each output joint from at most 4 vertices
        reg[torch.randint(V, (4,), generator=g), j] = torch.rand(4, generator=g) * 0.5
    return dict(v_template=_randn(g, V, 3, scale=0.3), shapedirs=_randn(g, nb, V * 3, scale=0.03 * blend),
                J_regressor=jr / jr.sum(0, keepdim=True), posedirs=_randn(g, SMPL_NPF, V * 3, scale=0.017 * blend),
                parents=np.array(SMPL_PARENTS, dtype=np.int32), weights=w / w.sum(1, keepdim=True), joint_regressor=reg)


def smpl_device_model(m):
    """The kernel's model dict: impersonator_b200.smpl.SMPL._device_model's folding of the joint regression."""
    V, nb = m["v_template"].shape[0], m["shapedirs"].shape[0]
    Jr = m["J_regressor"].double().t()
    js = torch.einsum('jv,kvd->jdk', Jr, m["shapedirs"].double().view(nb, V, 3)).reshape(72, nb)
    return dict(v_template=m["v_template"].contiguous(), shapedirs=m["shapedirs"].contiguous(),
                posedirs=m["posedirs"].contiguous(), weights=m["weights"].contiguous(),
                j_template=(Jr @ m["v_template"].double()).float().contiguous(), j_shapedirs=js.float().contiguous(),
                parents=torch.tensor(SMPL_PARENTS, dtype=torch.int32), joint_regressor_t=m["joint_regressor"].t().contiguous())


def smpl_bars(m, beta, theta, rotate_base, cam):
    """S of every smpl_forward output, in units of u: a first-order forward error analysis of the kernel's fp32
    operations, evaluated on the float64 values.

    Entrywise |.| products of the 9 rotations along a chain grow like 3^9, far above any real error, because a rotation
    does not grow an error vector.  So the chain is bounded in 2-norms: E_i bounds the spectral norm of the error of the
    global rotation of joint i, T_i the norm of the error of its translation.  Rotating an error keeps its norm, so
    along the chain E_i = E_parent + e_R(i) + 9 adds up.  Here e_R is 3x the largest entry bound of Rodrigues' error,
    and 9 is the 3x3 product's rounding (3-term dots of unit rows and columns).  So the bar grows linearly with the
    chain depth (at most 9 levels), not geometrically.  Each operation counts one u on the magnitudes it combines:
      Rodrigues  8 (|c| I + |1 - c| |r r^T| + |s| |[r]x| + angle + 1): the fp32 angle is a few ulps of itself off, and
                 cosf / sinf an ulp of 1
      joints J   nb + 2 on |J_reg|^T (|v_template| + |shapedirs|^T |beta|) (the folded fp32 regression, nb fma)
      v_posed    56 on |pf| |posedirs| (52 fma per K slice + the adds), nb + 3 on the shape blend and template
      skinning   24 + 4 on (|w| |A|) [|v_posed|; 1] (the 24-joint sum, then the 4-term product)
      joints     ceil(V / 128) + 7 on |reg|^T |verts| (128 thread-strided sums and a 7-level tree)
    SMPL_TAU = 2 leaves room for the second-order terms."""
    from oracle import smpl_ref
    d = lambda t: torch.as_tensor(t).double()                    # noqa: E731
    N, V, nb = beta.shape[0], m["v_template"].shape[0], beta.shape[1]
    vt, sd, pd, Jreg, W, reg = (d(m[k]) for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "weights",
                                                   "joint_regressor"))
    b = beta.double()
    t = theta.double().view(N, SMPL_NJ, 3)
    angle = torch.norm(t + 1e-8, dim=2, keepdim=True)
    r = t / angle
    c, s = torch.cos(angle)[..., None], torch.sin(angle)[..., None]
    ra = r.abs()
    skew = torch.stack([torch.zeros_like(ra[..., 0]), ra[..., 2], ra[..., 1], ra[..., 2], torch.zeros_like(ra[..., 0]),
                        ra[..., 0], ra[..., 1], ra[..., 0], torch.zeros_like(ra[..., 0])], dim=-1).view(N, SMPL_NJ, 3, 3)
    SR = 8 * (c.abs() * torch.eye(3, dtype=torch.float64) + (1 - c).abs() * ra[..., :, None] * ra[..., None, :]
              + s.abs() * skew + (angle + 1)[..., None])
    Rs = smpl_ref.rodrigues(t.reshape(-1, 3)).view(N, SMPL_NJ, 3, 3)
    v_shaped = (b @ sd).view(N, V, 3) + vt
    J = torch.stack([v_shaped[:, :, k] @ Jreg for k in range(3)], dim=2)                     # [N, 24, 3]
    SJ = torch.stack([((b.abs() @ sd.abs()).view(N, V, 3)[:, :, k] + vt.abs()[:, k]) @ Jreg.abs() for k in range(3)], dim=2)
    jerr = (nb + 2) * SJ.norm(dim=2)                                                        # [N, 24]
    pf = (Rs[:, 1:] - torch.eye(3, dtype=torch.float64)).reshape(N, SMPL_NPF)
    v_posed = (pf @ pd).view(N, V, 3) + v_shaped
    SV = (56 * (pf.abs() @ pd.abs()) + SR[:, 1:].reshape(N, SMPL_NPF) @ pd.abs()).view(N, V, 3) \
        + (nb + 3) * ((b.abs() @ sd.abs()).view(N, V, 3) + vt.abs())
    # the chain on true values, with E (rotation) and T (translation) error norms
    root = Rs[:, 0] @ torch.diag(torch.tensor([1., -1., -1.], dtype=torch.float64)) if rotate_base else Rs[:, 0]
    eR = 3 * SR.amax(dim=(2, 3))
    Gr, Gt, E, T = [root], [J[:, 0]], [eR[:, 0]], [jerr[:, 0]]
    for i in range(1, SMPL_NJ):
        p = SMPL_PARENTS[i]
        dJ = J[:, i] - J[:, p]
        tl = dJ.norm(dim=1)
        Gr.append(Gr[p] @ Rs[:, i])
        Gt.append((Gr[p] @ dJ[..., None])[..., 0] + Gt[p])
        E.append(E[p] + eR[:, i] + 9)
        T.append(T[p] + E[p] * tl + jerr[:, i] + jerr[:, p] + J[:, i].norm(dim=1) + J[:, p].norm(dim=1)
                 + 7 * (tl + Gt[p].norm(dim=1)))
    Gr, Gt, E, T = torch.stack(Gr, 1), torch.stack(Gt, 1), torch.stack(E, 1), torch.stack(T, 1)
    At = Gt - (Gr @ J[..., None])[..., 0]                                                   # A's translation column
    TA = T + E * J.norm(dim=2) + jerr + 7 * (J.norm(dim=2) + Gt.norm(dim=2))
    A_abs = torch.cat([Gr.abs(), At.abs()[..., None]], dim=3).reshape(N, SMPL_NJ, 12)
    skin = (W.abs()[None] @ A_abs).view(N, V, 3, 4)
    Sskin = (skin[..., :3] @ v_posed.abs()[..., None])[..., 0] + skin[..., 3]
    prop = (W[None] * E[:, None, :]).sum(-1) * v_posed.norm(dim=2) + (W[None] * TA[:, None, :]).sum(-1)
    S_verts = prop[..., None] + SV.norm(dim=2, keepdim=True) + 28 * Sskin
    verts = smpl_ref.forward(m, beta.double(), theta.double(), rotate_base=rotate_base)[0]
    rabs = reg.abs()
    S_joints = torch.stack([S_verts[:, :, k] @ rabs + ((V + 127) // 128 + 7) * (verts[:, :, k].abs() @ rabs)
                            for k in range(3)], dim=2)
    joints = torch.stack([verts[:, :, k] @ reg for k in range(3)], dim=2)
    cd = cam.double()
    S_j2d = cd[:, None, 0:1].abs() * (S_joints[..., :2] + 2 * (joints[..., :2].abs() + cd[:, None, 1:].abs()))
    return dict(verts=S_verts, joints=S_joints, Rs=SR, Jt=T[..., None].expand(N, SMPL_NJ, 3), j2d=S_j2d)


def _smpl(edge, seed, batch, V=33, nb=10, rotate_base=False, sparse=False, angles=None, wild=False, nan_joint=None):
    g = _gen(seed)
    m = smpl_model(seed, V, nb, sparse)
    beta = _randn(g, batch, nb)
    theta = _randn(g, batch, 72, scale=0.4)
    if wild:
        theta = (torch.rand(batch, 72, generator=g) * 2 - 1) * np.pi
    if angles is not None:                               # joint j of every frame at angles[j % len] about a random axis
        ax = _randn(g, batch, SMPL_NJ, 3).double()
        ax = ax / ax.norm(dim=2, keepdim=True)
        a = torch.tensor(angles, dtype=torch.float64)[torch.arange(SMPL_NJ) % len(angles)]
        theta = (ax * a[None, :, None]).float().reshape(batch, 72)
    if nan_joint is not None:                            # theta + 1e-8 = 0 in fp32: angle 0, r = -inf, the frame is NaN
        theta[batch // 2, nan_joint * 3:nan_joint * 3 + 3] = -1e-8
    cam = torch.cat([torch.rand(batch, 1, generator=g) + 0.5, _randn(g, batch, 2, scale=0.2)], dim=1)
    dm = smpl_device_model(m)
    built = {}

    def refs():                                          # built at the first check, not at import
        if not built:
            from oracle import smpl_ref
            verts, joints, Rs, Jt = smpl_ref.forward(m, beta.double(), theta.double(), rotate_base=rotate_base)
            ref = dict(verts=verts, joints=joints, Rs=Rs, Jt=Jt, j2d=smpl_ref.orth_proj_idrot(joints, cam.double()))
            if nan_joint is not None:                    # NaN exactly where the float32 oracle (the reference model) is NaN
                v32, j32, R32, J32 = smpl_ref.forward(m, beta, theta, rotate_base=rotate_base)
                r32 = dict(verts=v32, joints=j32, Rs=R32, Jt=J32, j2d=smpl_ref.orth_proj_idrot(j32, cam))
                ref = {k: torch.where(torch.isnan(r32[k].double()), float("nan"), v) for k, v in ref.items()}
            built["ref"] = ref
            built["S"] = smpl_bars(m, beta, theta, rotate_base, cam)
        return built

    def run(api, put, alloc):
        v, j, R, J, p = api.smpl_forward(put(beta), put(theta), {k: put(t) for k, t in dm.items()}, rotate_base=rotate_base,
                                         cam=put(cam))
        return dict(verts=v, joints=j, Rs=R, Jt=J, j2d=p)

    def tol(label, key, K):
        return Tol(label, key, lambda: refs()["ref"][key], lambda: refs()["S"][key], K, tau=SMPL_TAU)
    reg_terms = int((m["joint_regressor"] != 0).sum(0).max())
    case = Case("smpl_forward", edge, run, [tol("Rs", "Rs", 3), tol("J_transformed", "Jt", 4 * 9),
                                            tol("verts", "verts", SMPL_NPF + nb + SMPL_NJ), tol("joints", "joints", reg_terms),
                                            tol("j2d", "j2d", reg_terms + 1)], emulated=False)
    case.smpl = (m, beta, theta, rotate_base, cam, refs)
    return case


def smpl_cases():
    cases = [_smpl("batch=%d" % b, 1900 + b, b) for b in (1, 7, 8, 9, 16, 17)]
    cases += [
        _smpl("V=1", 1921, 3, V=1),
        _smpl("V=31 sparse weights", 1922, 3, V=31, sparse=True),
        _smpl("V=33 sparse weights", 1923, 9, V=33, sparse=True),
        _smpl("V=6890", 1924, 9, V=6890),
        _smpl("num_betas=1", 1925, 3, nb=1),
        _smpl("num_betas=16", 1926, 3, nb=16),
        _smpl("rotate_base", 1927, 9, rotate_base=True),
        _smpl("angles 0 1e-6 pi 2pi 3.5pi", 1928, 3, angles=[0.0, 1e-6, np.pi, 2 * np.pi, 3.5 * np.pi]),
        _smpl("wild poses", 1929, 9, wild=True, rotate_base=True),
        _smpl("NaN frame", 1930, 3, nan_joint=13),
    ]
    return cases


SMPL_EDGES = ["batch=%d" % b for b in (1, 7, 8, 9, 16, 17)] + [
    "V=1", "V=31 sparse weights", "V=33 sparse weights", "V=6890", "num_betas=1", "num_betas=16", "rotate_base",
    "angles 0 1e-6 pi 2pi 3.5pi", "wild poses", "NaN frame"]


from correspond_cases import CORRESPOND_EDGES, RASTER_EDGES, correspond_cases, raster_cases  # noqa: E402 (uses the above)

CASES = (norm_act_cases() + instance_stats_cases() + heads_cases() + frames_out_cases() + conv_direct_cases()
         + heads7x7_cases() + gated_bn_cases() + maxpool_cases() + avgpool_cases() + linear_cases() + lpips_cases()
         + layout_warp_cases() + attention_cases() + gated_cases() + smpl_cases() + correspond_cases() + raster_cases())

# The edges each front-end must be exercised at; one case each.
REQUIRED_EDGES = {
    "norm_act_nhwc": ["stats c=%d" % c for c in (8, 16, 64, 128, 256, 512, 1024, 2048)] + [
        "affine gamma+beta", "affine gamma only", "affine beta only", "bare", "stats relu residual", "bare warp",
        "EXT post affine res_step 2", "EXT res_step 2", "lo_format 1 c=512"] + [
        "warp sb=%s T %s ac=%d" % (sb, t, ac) for sb in ("1", "n") for t in ("same", "larger") for ac in (0, 1)] + [
        "range %s" % v for v in ("1023.7", "1023.75", "1024", "-1024", "59984", "59990", "60000", "65520", "+inf", "-inf",
                                 "nan")],
    "instance_stats_nhwc": ["hw=35 c=40", "hw=1000 c=96", "hw=16640 c=33"],
    "heads_composite": ["kw=%d w=%d c_stride=%d bg_batch=%s" % (kw, w, cs, b) for w in (1, 2, 3, 70)
                        for kw, cs, b in ((0, 4, "1"), (0, 32, "n"), (7, 32, "1"), (7, 32, "n"))] + [
        "u8 sweep", "range 8.0", "range below 8.0", "range -8.0", "range nan"],
    "frames_out": ["u8 sweep"],
    "conv2d_direct_nchw": ["cout=7", "dilation 2", "stride 2 odd sizes", "pad > k/2", "bias None", "1x1", "inpaintor 5x5",
                           "inpaintor 4x4 s2", "inpaintor 3x3 dil 16"],
    "conv7x7_heads_nhwc": ["1x1", "5x3", "17x65"],
    "gated_bn_nchw": ["act=%d %s" % (a, s) for a in (0, 1, 2) for s in ("no scale", "scale")],
    "maxpool_nchw_to_nhwc": ["112 -> 56 clipped last window", "h = k", "k < stride"],
    "global_avgpool_nhwc": ["scale relu ld_out > c", "no scale hw=1", "scale no relu"],
    "linear": ["k=1", "k=31 ld_x > k bias None", "k=85 m=1 ld_out > m", "k=2133", "accumulate into a slice"],
    "lpips_input": ["from01=0", "from01=1"],
    "lpips_layer": ["c=40 zero pixel layer 0", "hw=1 layer 2 accumulates"],
    "nhwc_to_nchw": ["c=4 c_stride=32", "c=100 hw=37x3"],
    "warp_nchw": ["accumulate src_batch=B C=70", "src_batch=1 T same size"],
    "self_attention_nhwc": ATTENTION_EDGES,
    "gated_act_nhwc": GATED_EDGES,
    "smpl_forward": SMPL_EDGES,
    "correspond": CORRESPOND_EDGES,
    "raster_forward_face_index_map": RASTER_EDGES,
}

# Front-ends the emulator replaces whose kernels are tested elsewhere: name -> "file::test function".
COVERED_ELSEWHERE = {
    "ConvPlan": "test_conv_gpu.py::test_conv2d",
    "pack_conv_weight": "test_conv_emulation_gpu.py::test_pack_conv_weight_bits",
    "pack_conv_weight_rowk": "test_conv_emulation_gpu.py::test_pack_conv_weight_rowk_bits",
    "nchw_to_nhwc_split": "test_conv_emulation_gpu.py::test_nchw_to_nhwc_split_bits",
    "pack_head_weights": "test_conv_gpu.py::test_heads_7x7",
    "det_bias_act": "test_detector_kernels_gpu.py::test_bias_act",
    "conv2d_direct_relu_nhwc": "test_metrics_gpu.py::test_stem_11x11_s4_matches_conv2d",
    "maxpool_nhwc": "test_metrics_gpu.py::test_floor_pool_nhwc_exact",
    "maxpool_nhwc_slice": "test_inception_gpu.py::test_maxpool_slice_exact",
    "bn_act_segment": "test_inception_gpu.py::test_bn_act_segment_matches_float64",
    "inception_input": "test_inception_gpu.py::test_input_matches_interpolate",
    "_correspond": "test_raster_gpu.py::test_correspond_matches_oracle",
    "frames_in": "test_frames_in_gpu.py::test_frames_in_matches_cv2_route",
}


def verify(case, outs, kernel):
    """Run the case's checks on CPU outputs; kernel=False skips the checks of kernel-only formats."""
    for chk in case.checks:
        if kernel or not chk.kernel_only:
            chk(case.name, outs)
