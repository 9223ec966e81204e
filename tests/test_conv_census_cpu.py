"""The census of conv-engine plans (tests/conv_census.py) on the CPU: the committed CENSUS is what the networks bind, every
census descriptor passes lwb_conv_plan_create's argument checks, and the windowed check of test_conv_census_gpu.py fails a
kernel that is wrong in one deliberate way."""
import pytest
import torch

import conv_census as C
from impersonator_b200 import kernels as K
from impersonator_b200._lib import ConvDesc
from test_conv_plan_cpu import L, create, has_device  # noqa: F401  (L, has_device: fixtures)


def test_census_matches_the_networks():
    """A network or binder change that adds or changes a plan must add its census case."""
    live = C.entries_of(C.live_census())
    committed = {e.name: e for e in C.CENSUS}
    changed = [e for e in live if committed.get(e.name) != e]
    gone = sorted(set(committed) - set(e.name for e in live))
    assert not changed and not gone, (
        "the networks bind plans CENSUS does not list (new or changed entries below), or CENSUS lists plans no network "
        "binds (%s).  The whole table, to paste into tests/conv_census.py:\n%s\nNew or changed:\n%s"
        % (gone, C.format_census(live), "".join(C.format_entry(e) for e in changed)))


def test_census_covers_every_kind():
    """The descriptor kinds the census exists for each appear as a case."""
    kinds = {
        "concat input on N = 128 tiles": lambda d, e: d["cin1"] and C.schedule(d)[0] == 128,
        "per-phase transposed conv with N = 128 tiles in fp16f8": lambda d, e: d["transposed"] == 1 and 2 in e.splits
        and C.schedule(d)[0] == 128,
        "merged transposed conv": lambda d, e: d["transposed"] == 2,
        "1x1 stride 2": lambda d, e: d["kh"] == d["kw"] == 1 and d["stride"] == 2,
        "odd count of 16-channel N tiles": lambda d, e: C.schedule(d)[0] == 16 and C.schedule(d)[4] % 2,
        "odd count of 64-channel N tiles": lambda d, e: C.schedule(d)[0] == 64 and C.schedule(d)[4] % 2,
        "cin 12544": lambda d, e: d["cin0"] == 12544,
        "100 images": lambda d, e: d["n"] == 100,
        "valid 3x3 on an odd size": lambda d, e: d["kh"] == 3 and d["pad"] == 0 and d["h_in"] % 2,
        "1x7 / 7x1 with pad_w": lambda d, e: (d["kh"], d["kw"]) in ((1, 7), (7, 1)) and d["pad_w"] >= 0,
        "row-K stem": lambda d, e: d["rowk"],
        "padded input channels": lambda d, e: e.cin_pad and e.cin_pad > C.real_dims(e)[0],
        "padded output channels": lambda d, e: e.cout_pad and e.cout_pad > C.real_dims(e)[1],
        "more than 15 tiles per CTA": lambda d, e: C.schedule(d)[6] > 15,
    }
    missing = [k for k, f in kinds.items() if not any(f(C.desc_of(e), e) for e in C.CENSUS)]
    assert not missing, missing


@pytest.mark.parametrize("entry", C.CENSUS, ids=[e.name for e in C.CENSUS])
def test_census_descriptor_passes_every_check(L, has_device, entry):  # noqa: F811
    for split in entry.splits:
        d = ConvDesc(w_exp=15, **dict(C.desc_of(entry), split=split))
        rc, err, plan = create(L, d)
        if not has_device:
            assert (rc, err) == (-2, "cuTensorMapEncodeTiled entry point not available"), (C.label(entry, split), err)
            continue
        assert rc == 0, (C.label(entry, split), err)
        L.lwb_conv_plan_destroy(plan)


# ---------------------------------------------------------------------------------------------------------------- teeth
# census entries at a reduced batch, one per tile orientation, plus a merged transposed conv: the "kernel output" is the
# float64 emulation of the whole output with exactly one deliberate change
TEETH = {
    "channel_major_concat": "conv3x3_s1_128+128_128_n1_128x128",        # N = 128, 16 x 8 tiles, statistics bound
    "swapped": "conv5x5_s1_64_64_n32_35x35_pw2",                         # N = 64, 32 x 8 tiles, partial, cin 48 of 64
    "pixel_major": "conv7x1_s1_64_32_n1_256x256_pw0_nt32",               # N = 32 (the folded heads)
    "merged": "convTm3x3_s2_128_64_n1_256x256",
}


def reduced(name, n=2):
    e = next(e for e in C.CENSUS if e.name == name)
    d = C.desc_of(e)
    n = min(n, d["n"])
    d["n"] = n
    return e._replace(desc=tuple(d[f] for f in C.DESC_FIELDS), x=(n,) + e.x[1:],
                      x1=(n,) + e.x1[1:] if e.x1 else None)


def case(kind):
    e = reduced(TEETH[kind])
    split = e.splits[0]
    x, w = C.make_inputs(e, seed=7)
    w_exp = K.weight_exponent(w.abs().max())
    out = C.emulated_output(e, x, w, split, w_exp)
    return e, split, x, w, w_exp, out


def sums(out):
    g = out.double().permute(0, 3, 1, 2)
    return torch.stack([g.sum(dim=(2, 3)), (g * g).sum(dim=(2, 3))], dim=-1)


@pytest.mark.parametrize("kind", list(TEETH))
def test_checker_passes_the_emulation(kind):
    e, split, x, w, w_exp, out = case(kind)
    C.check_output(e, split, x, w, w_exp, out, sums(out) if e.stats else None)


def _unwritten_column(e, split, x, w, w_exp, out):
    _, _, _, tx, _, _, _ = C.schedule(C.desc_of(e))
    out[:, :, (tx - 1) * C.TILE_W:] = float("nan")
    return x, w, out


def _shifted_row(e, split, x, w, w_exp, out):
    _, th, ty, _, _, _, _ = C.schedule(C.desc_of(e))
    y0 = (ty - 1) * th
    out[:, y0 + 1:] = out[:, y0:-1].clone()
    return x, w, out


def _concat_chunk_dropped(e, split, x, w, w_exp, out):
    d = C.desc_of(e)
    xm = x.clone()
    xm[:, d["cin0"]:d["cin0"] + 64] = 0
    return x, w, C.emulated_output(e, xm, w, split, w_exp)


def _tap_dropped(e, split, x, w, w_exp, out):
    wm = w.clone()
    wm[:, :, 3, 0] = 0
    return x, w, C.emulated_output(e, x, wm, split, w_exp)


def _phases_swapped(e, split, x, w, w_exp, out):
    a, b = out[:, 0::2, 1::2].clone(), out[:, 1::2, 0::2].clone()
    out[:, 0::2, 1::2], out[:, 1::2, 0::2] = b, a
    return x, w, out


def _padded_inputs_leak(e, split, x, w, w_exp, out):
    cin = C.real_dims(e)[0]
    extra = torch.randn((w.shape[0], x.shape[1] - cin) + tuple(w.shape[2:]), generator=torch.Generator().manual_seed(8))
    wl = torch.cat([w, extra * float(w.abs().max())], dim=1)
    leak = e._replace(weight=tuple(wl.shape))                          # a layer whose weights read the padded channels
    return x, w, C.emulated_output(leak, x, wl, split, K.weight_exponent(wl.abs().max()))


MUTANTS = {
    "last partial tile column unwritten": ("swapped", _unwritten_column, None),
    "last tile row shifted by one pixel": ("swapped", _shifted_row, None),
    "one K chunk of the concat's second input dropped": ("channel_major_concat", _concat_chunk_dropped, None),
    "one tap dropped": ("pixel_major", _tap_dropped, None),
    "two phase columns swapped": ("merged", _phases_swapped, None),
    "padded input channels leak": ("swapped", _padded_inputs_leak, None),
    "one tile's statistics missing": ("channel_major_concat", None, "stats"),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_checker_fails_the_mutant(mutant):
    kind, mutate, what = MUTANTS[mutant]
    e, split, x, w, w_exp, out = case(kind)
    st = sums(out) if e.stats else None
    if mutate is not None:
        x, w, out = mutate(e, split, x, w, w_exp, out)
        st = sums(out) if e.stats else None
    else:                                            # the first tile of image 0 never added its sums
        _, th, _, _, _, _, _ = C.schedule(C.desc_of(e))
        st[:1] -= sums(out[:1, :th, :C.TILE_W])
    with pytest.raises(C.CheckFailed) as failed:
        C.check_output(e, split, x, w, w_exp, out, st)
    print("%s: %s (err/bar %.3g)" % (mutant, failed.value, failed.value.ratio))
    assert failed.value.ratio > 4, str(failed.value)
