"""The bars of conv_emulation.check_conv discriminate: plausible kernel defects -- a correction product lost on one tap
group, on the last 64-channel K chunk or on the second concat input, one e4m3 product lost in fp16f8, one domain row
missing from or counted twice in the InstanceNorm statistics -- move the result by at least twice the bar that would
catch them.  The conv mutants move the output by about as much as the fp32 bars allow (2e-4 for fp16x3, 3e-4 for
fp16f8), which is why the conv tests compare against the emulation as well.  CPU only: the mutants are built from the
same float64 emulation on small shapes."""
import pytest
import torch
import torch.nn.functional as F

from conv_emulation import EMU_BAR, STATS_BAR, emulate, emulate_f8, f8_terms, split16, stats_errors
from impersonator_b200 import kernels as K


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def conv3(a, b):
    return F.conv2d(a, b, padding=1)


def distance(mutant, emu):
    return ((mutant - emu).abs().max() / emu.abs().max()).item()


def x3_mutant(x, w, drop, mask):
    """fp16x3 with the correction product ``drop`` (x_lo*w_hi or x_hi*w_lo) left out where ``mask`` (a 0/1 weight mask
    of w's shape) is 1."""
    E = K.weight_exponent(w.abs().max())
    emu = emulate(x, w, conv3, 1, E)
    xh, xl = split16(x)
    wh, wl = split16(w, 2.0 ** E)
    lost = conv3(xl, wh * mask) if drop == "x_lo*w_hi" else conv3(xh, wl * mask)
    return emu - lost / 2.0 ** E, emu


@pytest.mark.parametrize("drop", ["x_lo*w_hi", "x_hi*w_lo"])
def test_correction_dropped_on_one_tap_group(drop):
    """One filter column of a 3x3 filter (one y-halo tap group of three taps), 64 -> 64."""
    x, w = rnd(1, 64, 16, 16, seed=1), rnd(64, 64, 3, 3, seed=2, scale=0.05)
    mask = torch.zeros_like(w)
    mask[..., 0] = 1
    mut, emu = x3_mutant(x, w, drop, mask)
    d = distance(mut, emu)
    print("%s dropped on one tap group: %.3e (bar %.0e)" % (drop, d, EMU_BAR))
    assert d >= 2 * EMU_BAR


@pytest.mark.parametrize("drop", ["x_lo*w_hi", "x_hi*w_lo"])
def test_correction_dropped_on_last_k_chunk(drop):
    """128 -> 64: the second of two 64-channel K chunks."""
    x, w = rnd(1, 128, 16, 16, seed=3), rnd(64, 128, 3, 3, seed=4, scale=0.05)
    mask = torch.zeros_like(w)
    mask[:, 64:] = 1
    mut, emu = x3_mutant(x, w, drop, mask)
    d = distance(mut, emu)
    print("%s dropped on the last K chunk: %.3e (bar %.0e)" % (drop, d, EMU_BAR))
    assert d >= 2 * EMU_BAR


def test_correction_dropped_on_second_concat_input():
    """64 + 128 -> 64 skipper: x_lo*w_hi of the second tensor (both of its K chunks) left out."""
    a, b = rnd(1, 64, 16, 16, seed=5), rnd(1, 128, 16, 16, seed=6)
    w = rnd(64, 192, 3, 3, seed=7, scale=0.05)
    mask = torch.zeros_like(w)
    mask[:, 64:] = 1
    mut, emu = x3_mutant(torch.cat([a, b], dim=1), w, "x_lo*w_hi", mask)
    d = distance(mut, emu)
    print("second concat input's correction dropped: %.3e (bar %.0e)" % (d, EMU_BAR))
    assert d >= 2 * EMU_BAR


@pytest.mark.parametrize("half", ["x*w_lo", "x_lo*w"])
def test_fp16f8_e4m3_product_dropped(half):
    x, w = rnd(1, 64, 16, 16, seed=8), rnd(64, 64, 3, 3, seed=9, scale=0.05)
    E = K.weight_exponent(w.abs().max())
    main, t2, t3 = f8_terms(x, w, conv3, E)
    emu = emulate_f8(x, w, conv3, E)
    mut = main + (t3 if half == "x*w_lo" else t2)
    d = distance(mut, emu)
    print("fp16f8 without e4m3 %s: %.3e (bar %.0e)" % (half, d, EMU_BAR))
    assert d >= 2 * EMU_BAR


def tile_stats(got, chunk=256):
    """Statistics the way the epilogues form them: fp32 partial sums of at most ``chunk`` values (added in sequence, the
    worst order), then float64 sums of the partials."""
    n, c = got.shape[:2]
    v = got.float().reshape(n, c, -1)
    st = torch.zeros(n, c, 2, dtype=torch.float64)
    for p in range(0, v.shape[-1], chunk):
        part = v[..., p:p + chunk]
        st[..., 0] += part.cumsum(-1)[..., -1].double()
        st[..., 1] += (part * part).cumsum(-1)[..., -1].double()
    return st


@pytest.mark.parametrize("mutant", ["row_missing", "row_twice"])
def test_stats_row_missing_or_counted_twice(mutant):
    """A 20-row output (a partial second 16-row tile): statistics without the last domain row, or with it twice."""
    x, w = rnd(2, 64, 20, 12, seed=10), rnd(64, 64, 3, 3, seed=11, scale=0.05)
    got = emulate(x, w, conv3, 1, K.weight_exponent(w.abs().max())).float()
    st = tile_stats(got)
    e1, e2 = stats_errors(st, got)
    print("fp32 tile partials: sum %.3e sumsq %.3e (bar %.0e)" % (e1, e2, STATS_BAR))
    assert e1 <= STATS_BAR and e2 <= STATS_BAR                # the bar admits the epilogues' fp32 partial sums
    row = got[:, :, -1:].double()
    sign = -1.0 if mutant == "row_missing" else 1.0
    bad = st.clone()
    bad[..., 0] += sign * row.sum(dim=(2, 3))
    bad[..., 1] += sign * (row * row).sum(dim=(2, 3))
    e1, e2 = stats_errors(bad, got)
    print("%s: sum %.3e sumsq %.3e (bar %.0e)" % (mutant, e1, e2, STATS_BAR))
    assert max(e1, e2) >= 2 * STATS_BAR
