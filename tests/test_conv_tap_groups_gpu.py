"""Tap-group shapes of the conv engine that the layer tests do not reach: a filter column longer than one y-halo group
(split into two groups), dilated taps (groups of one) and a 4x4 stride-2 filter (two parity views with two-tap groups),
in the fp16x3 and fp16f8 operand modes, against float64 emulations of their arithmetic and torch fp32 on CPU."""
import pytest
import torch.nn.functional as F

from conv_emulation import check_conv
from test_conv_gpu import rnd, run_conv

pytestmark = pytest.mark.gpu

CASES = [
    # name, cin, cout, h, w, kh, kw, stride, pad, pad_w, dil
    ("9x1_column", 64, 64, 40, 24, 9, 1, 1, 4, 0, 1),
    ("3x3_dil2", 64, 64, 32, 32, 3, 3, 1, 2, None, 2),
    ("4x4_s2", 64, 128, 64, 64, 4, 4, 2, 1, None, 1),
]


@pytest.mark.parametrize("split", [1, 2])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_tap_groups(cuda, case, split):
    name, cin, cout, h, w, kh, kw, stride, pad, pad_w, dil = case
    x = rnd(2, cin, h, w, seed=41)
    wt = rnd(cout, cin, kh, kw, seed=42, scale=0.05)
    padding = (pad, pad if pad_w is None else pad_w)
    conv = lambda a, b: F.conv2d(a, b, stride=stride, padding=padding, dilation=dil)      # noqa: E731
    got, st, e = run_conv(cuda, x, wt, stride=stride, pad=pad, pad_w=pad_w, dil=dil, split=split)
    check_conv(name, split, got, x, wt, conv, e, st)


@pytest.mark.parametrize("split", [1, 2])
def test_conv_odd_m_tiles_many_rounds(cuda, split):
    """15 images of 40x24 = 135 M tiles (an odd count) x 2 N tiles: more tiles than CTAs of the persistent grid, so the
    tile loop and both operand rings wrap around across tiles."""
    x = rnd(15, 64, 40, 24, seed=43)
    wt = rnd(256, 64, 3, 3, seed=44, scale=0.05)
    conv = lambda a, b: F.conv2d(a, b, padding=1)      # noqa: E731
    got, st, e = run_conv(cuda, x, wt, pad=1, split=split)
    check_conv("odd_m", split, got, x, wt, conv, e, st)
