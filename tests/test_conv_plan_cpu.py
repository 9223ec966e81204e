"""lwb_conv_plan_create on every conv variant: each argument check with its return code and message, and how far a
valid descriptor gets.  A plan only encodes TMA descriptors from the buffer addresses, so aligned dummy pointers stand
in for the buffers and nothing is read or written.  Without a GPU the SM count falls back to 132, every check is
reached, and a valid descriptor stops at tensor-map encoding, which needs the driver; with a GPU the plan is built."""
import ctypes

import pytest
import torch

from impersonator_b200 import _lib
from impersonator_b200.kernels import make_conv_desc

PTRS = ("x0_hi", "x0_lo", "x1_hi", "x1_lo", "w_hi", "w_lo", "out_raw", "stats")


@pytest.fixture(scope="module")
def L():
    return _lib.lib()


def create(L, d, null=()):
    """lwb_conv_plan_create with a distinct 1 MB-aligned dummy address per buffer, NULL for the names in ``null``."""
    ptrs = [None if name in null else ctypes.c_void_p((i + 1) << 20) for i, name in enumerate(PTRS)]
    plan = ctypes.c_void_p()
    rc = L.lwb_conv_plan_create(ctypes.byref(d), *ptrs, ctypes.byref(plan))
    return rc, L.lwb_last_error().decode(), plan


def desc(kw):
    """make_conv_desc(**kw), then the struct fields in kw["fields"] set as given."""
    kw = dict(kw)
    fields = kw.pop("fields", {})
    d = make_conv_desc(**kw)
    for name, value in fields.items():
        setattr(d, name, value)
    return d


PLAIN = dict(n=2, h_in=32, w_in=32, cin0=64, cout=128, kh=3, kw=3, pad=1)
ROWK = dict(n=2, h_in=64, w_in=64, cin0=8, cout=64, kh=7, kw=7, pad=3, rowk=True, row_pitch=72)
STRIDE2 = dict(n=2, h_in=64, w_in=64, cin0=64, cout=128, kh=3, kw=3, stride=2, pad=1)
CONCAT = dict(PLAIN, cin1=128)
TRANSPOSED = dict(n=2, h_in=16, w_in=16, cin0=128, cout=64, kh=3, kw=3, stride=2, pad=1, transposed=True)
MERGED = dict(TRANSPOSED, fields=dict(transposed=2))

VALID = {
    "rowk": ROWK,
    "rowk_fp16": dict(ROWK, split=0),
    "rowk_halo": dict(ROWK, halo=True),
    "plain3x3": PLAIN,
    "plain3x3_fp16": dict(PLAIN, split=0),
    "plain3x3_f8": dict(PLAIN, split=2),
    "7x1_pad_w": dict(PLAIN, cout=64, kh=7, kw=1, pad=3, pad_w=0),
    "dilated": dict(PLAIN, pad=2, dil=2),
    "1x1": dict(PLAIN, kh=1, kw=1, pad=0),
    "stride2": STRIDE2,
    "stride2_f8": dict(STRIDE2, split=2),
    "stride2_7x7": dict(STRIDE2, cout=64, kh=7, kw=7, pad=3),
    "concat": CONCAT,
    "concat_f8": dict(CONCAT, split=2),
    "transposed": TRANSPOSED,
    "transposed_f8": dict(TRANSPOSED, split=2),
    "merged": MERGED,
    "merged_cout32": dict(MERGED, cout=32),
    "merged_f8": dict(MERGED, split=2),
    "halo3x3": dict(PLAIN, halo=True),
    "halo7x7": dict(PLAIN, cout=64, kh=7, kw=7, pad=3, halo=True),
    "halo1x9": dict(PLAIN, kh=1, kw=9, pad=0, pad_w=4, halo=True),
}
VALID.update({"n_tile%d" % nt: dict(PLAIN, cout=256, n_tile=nt) for nt in (16, 32, 64, 128, 256)})


@pytest.fixture(scope="module")
def has_device(L):
    """Whether a GPU is present.  If so, its context is made current: tensor maps are encoded within a context."""
    if L.lwb_device_info(None, None, None) != 0:
        return False
    torch.empty(1, device="cuda")
    return True


@pytest.mark.parametrize("name", list(VALID))
def test_valid_descriptor_passes_every_check(L, has_device, name):
    d = desc(VALID[name])
    rc, err, plan = create(L, d)
    if not has_device:
        assert (rc, err) == (-2, "cuTensorMapEncodeTiled entry point not available")
        assert not plan.value
        return
    assert rc == 0, err
    try:
        assert L.lwb_conv_plan_num_launches(plan) == (4 if d.transposed == 1 else 1)
    finally:
        L.lwb_conv_plan_destroy(plan)


CHECK = "lwb_conv_plan_create: "
# name -> (descriptor, NULL buffers, return code, message): one descriptor per check of lwb_conv_plan_create, in the
# order of the checks, each failing that check first
INVALID = {
    "null_pointer": (PLAIN, ("x0_hi",), -1, CHECK + "null pointer"),
    "split": (dict(PLAIN, split=3), (), -1, CHECK + "split must be 0, 1 or 2"),
    "lo_operands": (PLAIN, ("w_lo",), -1, CHECK + "split mode needs the lo operands"),
    "f8_rowk": (dict(ROWK, split=2), (), -1, CHECK + "the fp8 lo mode is not available for row-K / halo plans"),
    "f8_halo": (dict(PLAIN, split=2, halo=True), (), -1, CHECK + "the fp8 lo mode is not available for row-K / halo plans"),
    "size": (dict(PLAIN, n=0), (), -1, CHECK + "non-positive size"),
    "cout16": (dict(PLAIN, cout=40), (), -1, CHECK + "cout must be a multiple of 16"),
    "w_exp": (dict(PLAIN, fields=dict(w_exp=61)), (), -1, CHECK + "w_exp out of range"),
    "n_tile": (dict(PLAIN, cout=48, n_tile=32), (), -1, CHECK + "no N tile divides cout"),
    "halo_stride": (dict(STRIDE2, halo=True), (), -1, CHECK + "halo mode needs stride 1, dilation 1, not transposed"),
    "halo_transposed": (dict(TRANSPOSED, halo=True), (), -1, CHECK + "halo mode needs stride 1, dilation 1, not transposed"),
    "halo_rowk": (dict(ROWK, halo=True, row_pitch=64), (), -1, CHECK + "row-K shape"),
    "halo_even": (dict(PLAIN, kh=4, kw=4, halo=True), (), -1,
                  CHECK + "halo mode needs an odd kernel, kw <= 9, with 'same' padding (kh/2, kw/2)"),
    "rowk_stride": (dict(ROWK, stride=2), (), -1, CHECK + "row-K needs stride 1, kw <= 8, 8 channels"),
    "rowk_shape": (dict(ROWK, row_pitch=64), (), -1, CHECK + "row-K shape"),
    "cin": (dict(PLAIN, cin0=60), (), -1, CHECK + "input channels must be multiples of 64"),
    "second_input": (CONCAT, ("x1_hi",), -1, CHECK + "second input missing"),
    "second_input_lo": (CONCAT, ("x1_lo",), -1, CHECK + "second input missing"),
    "taps": (dict(PLAIN, kh=8, kw=8, pad=3), (), -1, CHECK + "too many filter taps"),
    "transposed_kernel": (dict(TRANSPOSED, pad=0), (), -1, CHECK + "transposed conv: only k3 s2 p1 op1"),
    "merged_kernel": (dict(MERGED, kh=1, kw=1), (), -1, CHECK + "transposed conv: only k3 s2 p1 op1"),
    "transposed_output": (dict(TRANSPOSED, fields=dict(h_out=34)), (), -1, CHECK + "transposed conv output must be 2x input"),
    "merged_output": (dict(MERGED, fields=dict(transposed=2, h_out=34)), (), -1, CHECK + "transposed conv output must be 2x input"),
    "merged_cout": (dict(MERGED, cout=48), (), -1, CHECK + "merged transposed conv needs cout in multiples of 32"),
    "stride": (dict(PLAIN, stride=3), (), -1, CHECK + "stride must be 1 or 2"),
    "stride2_concat": (dict(STRIDE2, cin1=64), (), -1, CHECK + "concat input only with stride 1"),
    "tap_offset": (dict(PLAIN, pad=130), (), -3, "conv_tc: tap offset out of range"),
}


@pytest.mark.parametrize("name", list(INVALID))
def test_invalid_descriptor_fails_its_check(L, name):
    kw, null, code, msg = INVALID[name]
    rc, err, plan = create(L, desc(kw), null)
    assert (rc, err) == (code, msg)
    assert not plan.value


def test_null_descriptor(L):
    plan = ctypes.c_void_p()
    rc = L.lwb_conv_plan_create(None, *[ctypes.c_void_p(1 << 20)] * 8, ctypes.byref(plan))
    assert (rc, L.lwb_last_error()) == (-1, b"lwb_conv_plan_create: null pointer")
    assert not plan.value
