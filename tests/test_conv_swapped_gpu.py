"""Plans with an N tile of 64 run the swapped orientation of the conv engine (64 output channels x 256-pixel tiles of
32 x 8, weights as the wgmma A operand).  Every kind of plan that reaches it, in the three operand modes -- fp16f8
(split 2), fp16x3 (split 1) and single-pass fp16 (split 0) -- against torch fp32 on CPU, with the bars of the layer tests:
partial 32-row tiles, concat inputs, the row-K stem, stride 2, the per-phase transposed conv, a forced N tile of 64 on
128 channels (two channel tiles) and an odd tile count larger than the persistent grid."""
import pytest
import torch
import torch.nn.functional as F

from conv_emulation import check_conv
from test_conv_gpu import rnd, run_conv, run_stem

pytestmark = pytest.mark.gpu

SPLITS = [2, 1, 0]


CASES = [
    # name, n, cin, cout, h, w, k, stride, n_tile
    ("ragged_40x24", 2, 64, 64, 40, 24, 3, 1, 0),       # second tile row: 8 of 32 rows, warpgroup 1 has none
    ("s2_64_64_72x56", 2, 64, 64, 72, 56, 3, 2, 0),      # stride 2 onto 64 channels, 36 x 28 outputs
    ("forced_n64_128", 2, 64, 128, 48, 40, 3, 1, 64),    # two channel tiles of 64
    ("5x5_64_64_44x20", 1, 64, 64, 44, 20, 5, 1, 0),     # 36-row boxes, partial tiles in y and x
]


@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv_swapped(cuda, case, split):
    name, n, cin, cout, h, w, k, stride, n_tile = case
    x = rnd(n, cin, h, w, seed=61)
    wt = rnd(cout, cin, k, k, seed=62, scale=0.05)
    conv = lambda a, b: F.conv2d(a, b, stride=stride, padding=k // 2)      # noqa: E731
    got, st, e = run_conv(cuda, x, wt, stride=stride, pad=k // 2, split=split, n_tile=n_tile)
    check_conv(name, split, got, x, wt, conv, e, st)


@pytest.mark.parametrize("split,cin1", [(2, 64), (1, 64), (0, 64), (1, 128)], ids=["2", "1", "0", "1-cin1_128"])
def test_conv_swapped_concat(cuda, split, cin1):
    """The 64+64 -> 64 skipper: K chunks from two tensors (and 64+128, where the second tensor has two K chunks)."""
    a, b = rnd(2, 64, 40, 24, seed=63), rnd(2, cin1, 40, 24, seed=64)
    wt = rnd(64, 64 + cin1, 3, 3, seed=65, scale=0.05)
    conv = lambda xx, ww: F.conv2d(xx, ww, padding=1)      # noqa: E731
    got, st, e = run_conv(cuda, a, wt, split=split, x1=b)
    check_conv("concat_64_%d" % cin1, split, got, torch.cat([a, b], dim=1), wt, conv, e, st)


@pytest.mark.parametrize("split", SPLITS)
def test_conv_swapped_transposed_phases(cuda, split):
    """ConvTranspose2d(k3, s2, p1, op1) to 64 channels as four per-phase launches on a 20 x 12 phase grid."""
    x = rnd(2, 128, 20, 12, seed=66)
    wt = rnd(128, 64, 3, 3, seed=67, scale=0.05)
    conv = lambda a, b: F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1)      # noqa: E731
    got, st, e = run_conv(cuda, x, wt, stride=2, pad=1, transposed=True, split=split)
    check_conv("convT_128_64", split, got, x, wt, conv, e, st)


@pytest.mark.parametrize("split", SPLITS)
def test_conv_swapped_odd_tiles_many_rounds(cuda, split):
    """15 images of 72x24 = 135 tiles of 32 x 8 (an odd count, more than the CTAs of the persistent grid), so the tile
    loop and both operand rings wrap around across tiles."""
    x = rnd(15, 64, 72, 24, seed=68)
    wt = rnd(64, 64, 3, 3, seed=69, scale=0.05)
    conv = lambda a, b: F.conv2d(a, b, padding=1)      # noqa: E731
    got, st, e = run_conv(cuda, x, wt, pad=1, split=split)
    check_conv("odd_tiles", split, got, x, wt, conv, e, st)


@pytest.mark.parametrize("split", [1, 0])
@pytest.mark.parametrize("size", [40, 72])
def test_stem_rowk_swapped(cuda, split, size):
    """The 7x7 stem (6 -> 64) through the row-K layout at sizes 32 does not divide (38-row boxes, partial last tile).
    The row-K plan has no fp8 path: fp16x3 is what the generator runs it in."""
    x = rnd(2, 6, size, size, seed=70)
    wt = rnd(64, 6, 7, 7, seed=71, scale=0.05)
    got, st, e = run_stem(cuda, x, wt, split)
    check_conv("stem_rowk_%d" % size, split, got, x, wt, lambda a, b: F.conv2d(a, b, padding=3), e, st)
