"""Error behaviour of the C ABI without a GPU: bad arguments are rejected with LWB_E_INVALID and a
message (the reference's CHECK_INPUT raises RuntimeError, rasterize_cuda.cpp:66-68) before any CUDA
call is made, so these run on the CPU-only box."""
import ctypes

import pytest

from impersonator_b200 import _lib


@pytest.fixture(scope="module")
def L():
    return _lib.lib()


def test_null_pointers_rejected(L):
    rc = L.lwb_raster_forward_face_index_map(None, 1, 1, 16, 0.1, 100.0, None, None, None, None, 0, None, None)
    assert rc == -1 and b"null pointer" in L.lwb_last_error()
    rc = L.lwb_warp_nchw(None, 1, 1, 4, 4, None, 1, 4, 4, 0, None, 0, None)
    assert rc == -1
    rc = L.lwb_norm_act_nhwc(None, None, None, None, 1e-5, 0, 1, 4, 4, 8, None, None, 0, None, 0, 0, 0, None, None, None, None, 0, None, None, 0, 1, None, None)
    assert rc == -1


def test_bad_sizes_rejected(L):
    dummy = ctypes.c_void_p(16)
    rc = L.lwb_raster_forward_face_index_map(dummy, 0, 5, 16, 0.1, 100.0, dummy, dummy, None, None, 0, dummy, None)
    assert rc == -1 and b"non-positive" in L.lwb_last_error()
    rc = L.lwb_correspond(dummy, dummy, dummy, 4, 10, 10, 16, 0.1, 100.0, 2.7, dummy, 3, dummy, None, 3, 0,
                          dummy, dummy, dummy, None, None, dummy, None)
    assert rc == -1 and b"src_batch" in L.lwb_last_error()
    rc = L.lwb_norm_act_nhwc(dummy, None, None, None, 1e-5, 0, 1, 4, 4, 12, None, None, 0, None, 0, 0, 0, None, None, None, None, 0, None, None, 0, 1, None, None)
    assert rc == -1 and b"multiple of 8" in L.lwb_last_error()
    rc = L.lwb_norm_act_nhwc(dummy, None, None, None, 1e-5, 0, 1, 4, 4, 32, None, None, 0, None, 0, 0, 0, None, None, dummy, dummy, 1, None, None, 0, 1, None, None)
    assert rc == -1 and b"blocks of 64" in L.lwb_last_error()
    assert L.lwb_raster_workspace_bytes(0, 256, 10) == 0
    assert L.lwb_raster_workspace_bytes(2, 256, 100) == 2 * 256 * 256 * 8 + 16 + 2 * 100 * 4


def test_direct_conv_rejects_an_empty_output(L):
    """h + 2p - d(k-1) - 1 in [-(s-1), -1]: floor division gives no output row, C's truncating division one."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("dummy pointers: an accepted call would launch on the visible GPU")
    dummy = ctypes.c_void_p(1024)
    # n, cin, h, w, cout, kh, kw, stride, pad, dil: 2 + 0 - 2 - 1 = -1 rows at stride 2, then the same for columns
    for h, w in ((2, 8), (8, 2)):
        rc = L.lwb_conv2d_direct_nchw(dummy, dummy, None, 1, 3, h, w, 4, 3, 3, 2, 0, 1, dummy, None)
        assert rc == -1 and b"empty output" in L.lwb_last_error(), (h, w, rc, L.lwb_last_error())
    rc = L.lwb_conv2d_direct_nchw(dummy, dummy, None, 1, 3, 8, 8, 4, 3, 3, 3, 0, 4, dummy, None)     # 8 - 8 - 1 = -1, dil 4
    assert rc == -1 and b"empty output" in L.lwb_last_error()


def test_conv_plan_argument_checks(L):
    d = _lib.ConvDesc(n=1, h_in=32, w_in=32, h_out=32, w_out=32, cin0=60, cin1=0, cout=64, kh=3, kw=3, stride=1, pad=1,
                      dil=1, transposed=0, split=1, rowk=0, row_pitch=0, n_tile=0, halo=0)
    dummy = ctypes.c_void_p(1024)
    plan = ctypes.c_void_p()
    rc = L.lwb_conv_plan_create(ctypes.byref(d), dummy, dummy, None, None, dummy, dummy, dummy, None, ctypes.byref(plan))
    assert rc == -1 and b"multiples of 64" in L.lwb_last_error()
    d.cin0, d.cout = 64, 60
    rc = L.lwb_conv_plan_create(ctypes.byref(d), dummy, dummy, None, None, dummy, dummy, dummy, None, ctypes.byref(plan))
    assert rc == -1 and b"multiple of 16" in L.lwb_last_error()
    d.cout = 64
    rc = L.lwb_conv_plan_create(ctypes.byref(d), dummy, None, None, None, dummy, None, dummy, None, ctypes.byref(plan))
    assert rc == -1 and b"lo operands" in L.lwb_last_error()
    assert L.lwb_conv_plan_run(None, None) == -1


def test_python_front_end_refuses_cpu_tensors():
    import torch
    from impersonator_b200 import kernels as K
    with pytest.raises(_lib.LwbError):
        K.warp_nchw(torch.zeros(1, 3, 8, 8), torch.zeros(1, 8, 8, 2))


def test_smpl_argument_checks(L):
    dummy = ctypes.c_void_p(1024)
    args = lambda **o: [o.get("beta", dummy), dummy, o.get("batch", 2), o.get("nb", 10), 6890, dummy, dummy, dummy, dummy, dummy,
                        dummy, dummy, o.get("reg", dummy), 19, 0, o.get("verts", dummy), o.get("joints", dummy), None, None,
                        o.get("cam", None), o.get("j2d", None), dummy, None]
    assert L.lwb_smpl_forward(*args(beta=None)) == -1 and b"null" in L.lwb_last_error()
    assert L.lwb_smpl_forward(*args(batch=0)) == -1 and b"positive" in L.lwb_last_error()
    assert L.lwb_smpl_forward(*args(nb=17)) == -1 and b"num_betas" in L.lwb_last_error()
    assert L.lwb_smpl_forward(*args(reg=None)) == -1 and b"regressor" in L.lwb_last_error()
    assert L.lwb_smpl_forward(*args(j2d=dummy)) == -1 and b"j2d" in L.lwb_last_error()
    assert L.lwb_smpl_workspace_bytes(0) == 0
    assert L.lwb_smpl_workspace_bytes(3) == 3 * (207 + 24 * 12) * 4
