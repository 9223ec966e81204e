"""Float64 emulations of the conv engine's three operand modes (DESIGN.md section 4) and the check every conv test runs.

Helper module for the conv tests, not a test file.  The emulations start from the fp32 ``x`` and ``w`` (not from the packed
bytes), so a packer that writes the wrong bits fails here as well as a kernel that multiplies the wrong ones:

* fp16 (split 0):   conv(x_hi, w_hi)
* fp16x3 (split 1): conv(x_hi, w_hi) + conv(x_hi, w_lo) + conv(x_lo, w_hi)
* fp16f8 (split 2): conv(x_hi, w_hi) + the two e4m3 correction products (``emulate_f8``)

with hi = fp16(v), lo = fp16(v - hi) (round to nearest even, subnormals included), the weights scaled by 2^w_exp before
the split and the result by 2^-w_exp, as the packers and the epilogue do.  What the kernel may still do differently is
the fp32 summation order of its accumulators.
"""
import numpy as np
import torch

from impersonator_b200 import kernels as K
from impersonator_b200.binding import RANGE_F8, RANGE_FP16

# max |got - emulation| / max |emulation|, every operand mode
EMU_BAR = 3e-5
# max |got - fp32 conv| / max |fp32 conv|, per operand mode
FP32_BAR = {0: 2e-2, 1: 2e-4, 2: 3e-4}
# |stats - sums of the kernel's own output| per (image, channel), relative to sum |got| (sum) and sum got^2 (sum of squares)
STATS_BAR = 2e-5


def report(name, got, ref):
    d = (got.double() - ref.double()).abs()
    scale = ref.abs().max().item() + 1e-30
    idx = np.unravel_index(int(d.argmax()), d.shape)
    print("%s: max-abs %.3e (ref scale %.3e, rel %.3e) at %s; mean-abs %.3e; nonfinite %d"
          % (name, d.max().item(), scale, d.max().item() / scale, idx, d.mean().item(),
             int((~torch.isfinite(got)).sum())))
    return d.max().item() / scale


# ------------------------------------------------------------------------------- operand formats (csrc/operands.cuh)
def fp16_pair(v):
    """The fp16 hi / lo split of fp32 v: hi = fp16(v), lo = fp16(v - hi)."""
    hi = v.half()
    return hi, (v - hi.float()).half()


def e4m3(t):
    """e4m3 with saturation at +-448 (__NV_SATFINITE)."""
    return t.clamp(-448, 448).to(torch.float8_e4m3fn)


def pair_blocks(a, b):
    """[..., C] e4m3 operands a, b -> [..., 2C] bytes: per 64-channel block, 64 bytes of a then 64 bytes of b."""
    lead, c = a.shape[:-1], a.shape[-1]
    blk = torch.stack([e4m3(a).view(torch.uint8).view(*lead, c // 64, 64),
                       e4m3(b).view(torch.uint8).view(*lead, c // 64, 64)], dim=-2)
    return blk.reshape(*lead, 2 * c)


def act_pair_blocks(v, hi=None):
    """The activation pair blocks (lo_format 1) of fp32 v [..., C] with its fp16 hi: e4m3(v / 16), e4m3((v - hi) * 1024)."""
    hi = v.half() if hi is None else hi
    return pair_blocks(v / 16, (v - hi.float()) * 1024)


def range_bits(hi):
    """The operand-range flag bits of an fp16 hi tensor."""
    a = hi.float().abs()
    if bool(((a >= 60000) | torch.isnan(a)).any()):
        return RANGE_F8 | RANGE_FP16
    return RANGE_F8 if bool((a >= 1024).any()) else 0


# an emitted value, its label and the range bits wanted: fp16 of 1023.7 -> 1023.5, 1023.75 -> 1024 (tie to even),
# 59983 / 59984 -> 59968 (tie to even), 59990 -> 60000 = 0x7b53, 65520 -> inf
RANGE_VALUES = (("1023.7", 1023.7, 0), ("1023.75", 1023.75, 1), ("1024", 1024.0, 1), ("-1024", -1024.0, 1),
                ("59984", 59984.0, 1), ("59990", 59990.0, 3), ("60000", 60000.0, 3), ("65520", 65520.0, 3),
                ("+inf", float("inf"), 3), ("-inf", float("-inf"), 3), ("nan", float("nan"), 3))


def to_f8_operands(cuda, x):
    """NCHW fp32 -> (hi fp16 NHWC, fp8 pair blocks) through the norm kernel used as a plain converter."""
    raw = x.permute(0, 2, 3, 1).contiguous().to(cuda)
    hi = torch.empty(raw.shape, dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    K.norm_act_nhwc(raw, None, None, None, False, None, y_hi=hi, y_lo=lo, lo_format=1)
    return hi, lo


# ------------------------------------------------------------------------------------------------------ emulations
def split16(v, scale=1.0):
    """(hi, lo) of v * scale as float64 tensors: hi = fp16(v * scale), lo = fp16(v * scale - hi).  v * scale is formed in
    fp32 (exact for a power-of-two scale), like the packers do."""
    hi, lo = fp16_pair(v.float() * scale)
    return hi.double(), lo.double()


def q8(t):
    """e4m3 with saturation at +-448 (__NV_SATFINITE), as float64."""
    return e4m3(t).double()


def f8_terms(x, w, conv, w_exp):
    """The three products of the fp16f8 mode, each already scaled back by 2^-E: x_hi*w_hi on the fp16 path,
    e4m3(x / 16) * e4m3(w_lo * 2^(E+4)) and e4m3(x_lo * 2^10) * e4m3(w * 2^(E-10)) on the fp8 path."""
    E = w_exp
    xh = x.half().double()
    wh = w.half().double()
    xl, wl = x.double() - xh, w.double() - wh
    main = conv(xh, wh)
    t2 = conv(q8(x.float() / 16), q8((wl * 2.0 ** (E + 4)).float())) / 2.0 ** E
    t3 = conv(q8((xl * 1024).float()), q8(w.float() * 2.0 ** (E - 10))) / 2.0 ** E
    return main, t2, t3


def emulate_f8(x, w, conv, w_exp=None):
    """The arithmetic the fp16f8 mode is meant to perform (DESIGN.md section 4), in float64: per-layer weight scale 2^E
    with max|w| * 2^E in [2^14, 2^15); x8 = e4m3(x / 16), xlo8 = e4m3(x_lo * 2^10), wlo8 = e4m3(w_lo * 2^(E+4)),
    w8 = e4m3(w * 2^(E-10))."""
    if w_exp is None:
        w_exp = K.weight_exponent(w.abs().max())
    main, t2, t3 = f8_terms(x, w, conv, w_exp)
    return main + t2 + t3


def emulate(x, w, conv, split, w_exp):
    """float64 result of ``conv`` in operand mode ``split`` (0 fp16, 1 fp16x3, 2 fp16f8) on fp32 x, w."""
    split = int(split)
    if split == 2:
        return emulate_f8(x, w, conv, w_exp)
    s = 2.0 ** w_exp
    xh, xl = split16(x)
    wh, wl = split16(w, s)
    y = conv(xh, wh)
    if split == 1:
        y = y + conv(xh, wl) + conv(xl, wh)
    return y / s


def stats_errors(st, got):
    """Per-(image, channel) errors of conv statistics st [n, c, 2] against float64 sums of the kernel's own NCHW output,
    relative to sum |got| and sum got^2."""
    g = got.double()
    s, a, q = g.sum(dim=(2, 3)), g.abs().sum(dim=(2, 3)), (g * g).sum(dim=(2, 3))
    st = st.double()
    e1 = (st[..., 0] - s).abs() / a.clamp(min=1e-300)
    e2 = (st[..., 1] - q).abs() / q.clamp(min=1e-300)
    return e1.max().item(), e2.max().item()


def check_stats(st, got):
    e1, e2 = stats_errors(st, got)
    print("stats vs the output's own sums: sum %.3e sumsq %.3e (bar %.0e)" % (e1, e2, STATS_BAR))
    assert e1 <= STATS_BAR and e2 <= STATS_BAR


BAND = 1 << 18                  # bytes of sentinel before and after each view (a multiple of 256: the views stay aligned)
SENTINEL = 0xA5


def guarded(cuda, shape, dtype, fill):
    """A contiguous ``shape`` view of ``dtype`` inside a byte buffer with BAND sentinel bytes on each side."""
    nbytes = torch.Size(shape).numel() * torch.empty((), dtype=dtype).element_size()
    buf = torch.full((BAND + nbytes + BAND,), SENTINEL, dtype=torch.uint8, device=cuda)
    view = buf[BAND:BAND + nbytes].view(dtype).view(shape)
    view.fill_(fill)
    return buf, view


def assert_bands_intact(name, buf):
    for side, band in (("before", buf[:BAND]), ("after", buf[-BAND:])):
        bad = (band != SENTINEL).nonzero()
        assert bad.numel() == 0, "%s: %d sentinel bytes %s the view were overwritten (first at %d)" % (
            name, bad.numel(), side, int(bad[0]) if bad.numel() else -1)


def check_conv(name, split, got, x, w, conv, w_exp, stats=None, emu_bar=EMU_BAR):
    """The checks of one conv-engine result ``got`` (NCHW fp32, CPU) of ``conv(x, w)`` in operand mode ``split``:
    (a) against the mode's float64 emulation, (b) against fp32, (c) the statistics against ``got`` itself."""
    split = int(split)
    mode = {0: "fp16", 1: "fp16x3", 2: "fp16f8"}[split]
    emu = emulate(x, w, conv, split, w_exp)
    assert report("%s/%s vs emulation" % (name, mode), got, emu) < emu_bar
    assert report("%s/%s vs fp32" % (name, mode), got, conv(x, w)) < FP32_BAR[split]
    if stats is not None:
        check_stats(stats, got)
