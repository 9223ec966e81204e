"""Every ``--map_name`` without a GPU: the generator width each map asks for, the stem padding it gets, the conv plan
checks of the row-K stem over 8 / 16 / 24 padded channels, the tables mesh.create_mapping builds, and the wide-map
generator golden (tests/golden/generator_wide.npz) held against oracle/generator_ref.py."""
import ctypes
import types

import numpy as np
import pytest
import torch

import generator_wide_cases as W
from impersonator_b200 import _lib, mesh
from impersonator_b200._lib import LwbError
from impersonator_b200.generator import STEM_MAX_CIN, stem_cin_pad
from impersonator_b200.imitator import Imitator
from impersonator_b200.kernels import make_conv_desc
from oracle import generator_ref as G

# map_name -> (conditioning channels, generator input channels src_dim = tsf_dim, padded stem channels)
MAPS = {"seg": (1, 4, 8), "ids": (1, 4, 8), "uv": (2, 5, 8), "uv_seg": (3, 6, 8), "par": (11, 14, 16),
        "binary": (15, 18, 24)}


@pytest.mark.parametrize("map_name", sorted(MAPS))
def test_cond_nc_and_generator_width(map_name):
    nc, src_dim, c_pad = MAPS[map_name]
    assert mesh.get_map_fn_dim(map_name) == nc
    im = types.SimpleNamespace(_opt=types.SimpleNamespace(map_name=map_name))
    assert Imitator.cond_nc(im) == (nc, nc)
    assert 3 + nc == src_dim and stem_cin_pad(src_dim) == c_pad


def test_stem_refuses_more_than_24_channels():
    assert STEM_MAX_CIN == 24 and stem_cin_pad(24) == 24 and stem_cin_pad(9) == 16
    for cin in (25, 32, 0):
        with pytest.raises(LwbError, match="the 7x7 stem takes 1 to 24 input channels, not %d" % cin):
            stem_cin_pad(cin)


def create(d):
    """lwb_conv_plan_create on dummy 1 MB-aligned buffers: -> (return code, error message)."""
    L = _lib.lib()
    ptrs = [ctypes.c_void_p((i + 1) << 20) for i in range(8)]
    plan = ctypes.c_void_p()
    rc = L.lwb_conv_plan_create(ctypes.byref(d), *ptrs, ctypes.byref(plan))
    err = L.lwb_last_error().decode()
    if plan.value:
        L.lwb_conv_plan_destroy(plan)
    return rc, err


def stem_desc(cin0, **kw):
    return make_conv_desc(2, 64, 64, cin0, 64, 7, kw.pop("kw", 7), pad=3, rowk=True, row_pitch=72, **kw)


@pytest.mark.parametrize("halo", [False, True])
@pytest.mark.parametrize("cin0", [8, 16, 24])
def test_wide_stem_plan_passes_every_check(cin0, halo):
    rc, err = create(stem_desc(cin0, halo=halo))
    if L_has_device():
        assert rc == 0, err
    else:
        assert (rc, err) == (-2, "cuTensorMapEncodeTiled entry point not available")


@pytest.mark.parametrize("cin0", [12, 32, 64])
def test_wide_stem_plan_refuses_other_channel_counts(cin0):
    assert create(stem_desc(cin0)) == (-1, "lwb_conv_plan_create: row-K needs 8, 16 or 24 padded input channels in one "
                                           "input")
    assert create(stem_desc(cin0, halo=True)) == (-1, "lwb_conv_plan_create: row-K shape")


def test_wide_stem_plan_refuses_wide_filters():
    assert create(stem_desc(24, kw=9)) == (-1, "lwb_conv_plan_create: row-K needs stride 1, kw <= 8, 8 channels")


def L_has_device():
    return _lib.lib().lwb_device_info(None, None, None) == 0


def test_ids_and_binary_tables(tmp_path):
    """'ids' stacks as one column (the face index / F, background -1); 'binary' codes the face index in 15 bits, the
    width the generator is built for, with an all -1 background row."""
    from impersonator_b200 import synthetic as S
    S.write_synthetic_assets(str(tmp_path))
    mp = str(tmp_path / "assets" / "pretrains" / "mapper.txt")
    nf = S.SMPL_F
    ids = mesh.create_mapping('ids', mp, contain_bg=True)
    assert ids.shape == (nf + 1, 1) and ids[-1, 0] == -1
    assert np.array_equal(ids[:nf, 0], np.arange(0, 1, 1 / nf, dtype=np.float32)[:nf])
    binary = mesh.create_mapping('binary', mp, contain_bg=True)
    assert binary.shape == (nf + 1, mesh.get_map_fn_dim('binary'))
    weights = 2 ** np.arange(14, -1, -1)
    assert np.array_equal(binary[:nf] @ weights, np.arange(nf)) and (binary[-1] == -1).all()
    for name in ("seg", "uv", "uv_seg", "par"):
        assert mesh.create_mapping(name, mp, contain_bg=True).shape == (nf + 1, mesh.get_map_fn_dim(name))


@pytest.fixture(scope="module")
def golden():
    torch.set_grad_enabled(False)
    return np.load(W.GOLD)


# the oracle on other machines (thread counts, oneDNN kernels) against slices made by the reference modules
ORACLE_TOL = 2e-4


@pytest.mark.parametrize("cin", W.WIDTHS)
def test_oracle_matches_wide_golden(golden, cin):
    g, p = golden, "w%d_" % cin
    _, sd = W.weights(cin)
    c = W.cases(cin)
    got = {}
    src = c["front"]["src"]
    got["stem_raw"] = W.stem_slice(torch.nn.functional.conv2d(src, sd["src_model.encoders.0.0.weight"], padding=3))
    enc, res = G.encode_src(src, sd)
    for i in range(4):
        got["enc%d" % i] = W.feat(enc[i])
    got["res5"] = W.feat(res[5])
    f = c["front"]
    for name, t in zip(("src_img", "src_mask", "tsf_img", "tsf_mask"), G.infer_front(f["src"], f["tsf"], f["T"], sd)):
        got["front_" + name] = W.sl(t)
    i2 = c["inf"]
    e, r = G.encode_src(i2["src"], sd)
    img, mask = G.inference(e, r, i2["tsf"], i2["T"], sd)
    got["inf_img"], got["inf_mask"] = W.sl(img), W.sl(mask)
    a, b = c["swap_a"], c["swap_b"]
    o12, q12 = G.encode_src(a["src"], sd)
    o21, q21 = G.encode_src(b["src"], sd)
    s_img, s_mask = G.swap(a["tsf"], o12, o21, q12, q21, a["T"], b["T"], sd)
    got["swap_img"], got["swap_mask"] = W.sl(s_img), W.sl(s_mask)
    keys = sorted(k[len(p):] for k in g.files if k.startswith(p) and not k.startswith(p + "512"))
    assert sorted(got) == keys
    for k in keys:
        d = float(np.abs(got[k] - g[p + k]).max())
        print("w%d %-14s oracle vs reference golden %.2e" % (cin, k, d))
        assert d < ORACLE_TOL, k
