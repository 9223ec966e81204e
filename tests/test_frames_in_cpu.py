"""The input path's arithmetic without a GPU: the numpy restatement of cv2's uint8 INTER_LINEAR resize (frames_in_cases)
against the cv2 installed here, the float step against numpy, and lwb_frames_in's argument checks."""
import ctypes

import numpy as np
import pytest

import frames_in_cases as F
from impersonator_b200 import _lib

cv2 = pytest.importorskip("cv2")


@pytest.mark.parametrize("h,w,size", F.SWEEP)
def test_restatement_equals_cv2_resize(h, w, size):
    img = F.frames(1, h, w, seed=h * 7919 + w * 31 + size)[0]
    for s in (size, F.HMR_SIZE):
        ref = cv2.resize(img, (s, s))
        got = F.resize_u8(img, s)
        assert got.shape == ref.shape
        n_bad = int((got != ref).sum())
        assert n_bad == 0, "%dx%d -> %d: %d bytes differ from cv2.resize" % (h, w, s, n_bad)


def test_restatement_on_a_4096_source():
    img = F.frames(1, 4096, 4096, seed=4)[0]
    for s in (256, 224):
        assert np.array_equal(F.resize_u8(img, s), cv2.resize(img, (s, s)))


def test_vertical_rounding_is_the_vector_one():
    """The textbook rounding (H0*b0 + H1*b1 + 2^21) >> 22 is not what cv2 computes: the sweep would not catch a
    restatement that used it on frames where both agree, so check that they disagree on a real frame."""
    img = F.frames(1, 333, 517, seed=1)[0]
    h, w, _ = img.shape
    x0, x1, a0, a1 = F.coefficients(w, 256, True)
    y0, y1, b0, b1 = F.coefficients(h, 256, False)
    rows = img.astype(np.int64)[:, x0] * a0[None, :, None] + img.astype(np.int64)[:, x1] * a1[None, :, None]
    scalar = np.clip((rows[y0] * b0[:, None, None] + rows[y1] * b1[:, None, None] + (1 << 21)) >> 22, 0, 255)
    ref = cv2.resize(img, (256, 256))
    assert (scalar != ref).sum() > 1000 and np.array_equal(F.resize_u8(img, 256), ref)


def test_float_step_equals_numpy():
    v = np.arange(256, dtype=np.uint8)
    ref = v.astype(np.float32) / 255.0 * 2 - 1.0
    got = F.kernel_float_steps(v)
    assert ref.dtype == np.float32 and np.array_equal(got.view(np.int32), ref.view(np.int32))
    assert np.array_equal(F.to_signed(v).view(np.int32), ref.view(np.int32))


def test_cv2_route_matches_restatement():
    frame = F.frames(1, 333, 517, seed=8)[0]
    img, hmr, gt = F.cv2_route(frame, 256)
    rgb = frame[..., ::-1]
    assert np.array_equal(img, F.to_signed(F.resize_u8(np.ascontiguousarray(rgb), 256)).transpose(2, 0, 1))
    assert np.array_equal(hmr, F.to_signed(F.resize_u8(np.ascontiguousarray(rgb), 224)).transpose(2, 0, 1))
    assert np.array_equal(gt, F.resize_u8(frame, 256))


@pytest.fixture(scope="module")
def L():
    return _lib.lib()


def test_frames_in_argument_checks(L):
    d = ctypes.c_void_p(1024)

    def call(frames=d, n=1, h=8, w=8, bgr=1, size=4, img=d, hmr_size=224, hmr=None, u8=None):
        return L.lwb_frames_in(frames, n, h, w, bgr, size, img, hmr_size, hmr, u8, None)

    for kw, msg in ((dict(frames=None), b"null frames"),
                    (dict(img=None), b"no output"),
                    (dict(n=0), b"non-positive"), (dict(h=0), b"non-positive"), (dict(w=-3), b"non-positive"),
                    (dict(size=0), b"non-positive size"), (dict(size=-1, img=None, u8=d), b"non-positive size"),
                    (dict(hmr=d, hmr_size=0), b"non-positive hmr_size"),
                    (dict(n=70000), b"65535"),
                    (dict(n=65535, h=2 ** 30, w=2 ** 30), b"overflows"),
                    (dict(size=2 ** 30), b"overflows")):
        rc = call(**kw)
        assert rc == -1 and msg in L.lwb_last_error(), (kw, rc, L.lwb_last_error())


def test_frame_stack_refuses_mixed_sizes_and_dtypes():
    from impersonator_b200.imitator import _frame_stack
    with pytest.raises(_lib.LwbError, match="one size"):
        _frame_stack([np.zeros((4, 4, 3), np.uint8), np.zeros((4, 5, 3), np.uint8)])
    with pytest.raises(_lib.LwbError, match="uint8"):
        _frame_stack(np.zeros((2, 4, 4, 3), np.float32))
    with pytest.raises(_lib.LwbError, match="uint8"):
        _frame_stack(np.zeros((2, 4, 4), np.uint8))
    assert _frame_stack([np.ones((4, 5, 3), np.uint8)] * 3).shape == (3, 4, 5, 3)


def test_a_16_bit_png_is_refused_naming_the_file(tmp_path, monkeypatch):
    """A 16-bit PNG decodes to uint16, which the reference's float conversion would scale to values up to 513: the
    Imitator raises before anything is computed, naming the file."""
    import kernel_emulator
    import tasks_common as C
    from impersonator_b200 import synthetic as S
    from impersonator_b200.generator import ImpersonatorGenerator
    from impersonator_b200.imitator import Imitator
    from impersonator_b200.nmr import SMPLRenderer
    kernel_emulator.install_tasks(monkeypatch)
    v, f = S.uv_sphere()
    path = str(tmp_path / "deep.png")
    assert cv2.imwrite(path, F.frames(1, 40, 30, seed=5)[0].astype(np.uint16) * 257)
    assert cv2.imread(path, -1).dtype == np.uint16
    render = SMPLRenderer(image_size=C.SIZE, faces=f.numpy(), map_fn=S.synthetic_tables()["map_fn"])
    im = Imitator(C.Opt(), generator=ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6),
                  hmr=S.QuarterTurnBodyModel(v), render=render, device="cpu")
    with pytest.raises(_lib.LwbError, match="deep.png decodes to uint16"):
        im.personalize(path, src_smpl=np.zeros(85, np.float32))
    with pytest.raises(_lib.LwbError, match="deep.png decodes to uint16"):
        im.transfer_params(path, tgt_smpl=np.zeros(85, np.float32))
