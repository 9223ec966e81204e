"""The input path on the GPU: lwb_frames_in against the cv2 route byte for byte over the sweep of frames_in_cases, and
Imitator / Viewer / Swapper driven by uint8 frames against the same classes driven by PNG files of those frames."""
import os

import numpy as np
import pytest
import torch

import frames_in_cases as F
import tasks_common as C
from impersonator_b200 import kernels as K
from impersonator_b200 import synthetic as S
from impersonator_b200._lib import LwbError
from impersonator_b200.generator import ImpersonatorGenerator
from impersonator_b200.imitator import Imitator
from impersonator_b200.nmr import SMPLRenderer
from impersonator_b200.swapper import Swapper
from impersonator_b200.viewer import Viewer

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def _bits(a):
    a = a.cpu().numpy() if torch.is_tensor(a) else a
    return a.view(np.int32) if a.dtype == np.float32 else a


@pytest.mark.parametrize("bgr", [True, False])
@pytest.mark.parametrize("batch", [1, 5])
@pytest.mark.parametrize("h,w,size", F.SWEEP)
def test_frames_in_matches_cv2_route(cuda, h, w, size, bgr, batch):
    fr = F.frames(batch, h, w, seed=h * 131 + w * 7 + size + batch)
    img, hmr, u8 = K.frames_in(torch.from_numpy(fr).to(cuda), size, bgr=bgr, want_img=True, want_hmr=True, want_u8=True)
    torch.cuda.synchronize()
    for i in range(batch):
        r_img, r_hmr, r_u8 = F.cv2_route(fr[i], size, bgr=bgr)
        assert np.array_equal(_bits(img[i]), _bits(r_img)), (h, w, size, bgr, i, "img")
        assert np.array_equal(_bits(hmr[i]), _bits(r_hmr)), (h, w, size, bgr, i, "hmr")
        assert np.array_equal(u8[i].cpu().numpy(), r_u8), (h, w, size, bgr, i, "u8")


def test_frames_in_subsets_and_host_sources(cuda):
    fr = F.frames(3, 333, 517, seed=3)
    full = K.frames_in(torch.from_numpy(fr).to(cuda), 256, want_img=True, want_hmr=True, want_u8=True)
    for src in (fr, torch.from_numpy(fr), list(fr)[0]):                       # numpy, host tensor, one [H,W,3] frame
        for want in ((True, False, False), (False, True, False), (False, False, True), (True, True, True)):
            got = K.frames_in(src, 256, want_img=want[0], want_hmr=want[1], want_u8=want[2])
            for g, f, on in zip(got, full, want):
                assert (g is None) != on
                if on:
                    assert torch.equal(g, f[:g.shape[0]])
    with pytest.raises(LwbError, match="no output"):
        K.frames_in(fr, 256, want_img=False, want_hmr=False, want_u8=False)
    with pytest.raises(LwbError, match="uint8"):
        K.frames_in(torch.zeros(2, 8, 8, 3, device=cuda), 256)


# ---- the task classes ----------------------------------------------------------------------------------------------

class RecordingHMR(object):
    """An HMR stand-in that keeps every input batch it is given and derives each frame's pose from its pixels
    (quarter turns of the exact QuarterTurnBodyModel body, so both routes rasterize identical vertices)."""

    def __init__(self, base_verts):
        self.body = S.QuarterTurnBodyModel(base_verts)
        self.inputs = []

    def __call__(self, img):
        self.inputs.append(img.detach().cpu().clone())
        theta = torch.zeros(img.shape[0], 85, device=img.device)
        theta[:, 0] = 0.9
        theta[:, 3] = torch.floor((img.mean(dim=(1, 2, 3)) + 1) * 64) % 4
        return theta

    def get_details(self, theta):
        return self.body.get_details(theta)


@pytest.fixture(scope="module")
def world(cuda, tmp_path_factory):
    torch.set_grad_enabled(False)
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    root = tmp_path_factory.mktemp("frames_in")
    frames = F.frames(5, 333, 517, seed=11)
    paths = []
    for i, fr in enumerate(frames):
        p = str(root / ("frame_%d.png" % i))
        cv2.imwrite(p, fr)
        assert np.array_equal(cv2.imread(p, -1), fr)                           # PNG: the file holds exactly the frame
        paths.append(p)
    return dict(v=v, f=f, tabs=tabs, net=net.to(cuda).eval(), frames=frames, paths=paths, root=root)


def _render(w, size):
    return SMPLRenderer(image_size=size, faces=w["f"].numpy(), map_fn=w["tabs"]["map_fn"])


def _opt(size=C.SIZE):
    opt = C.Opt()
    opt.image_size, opt.batch_size = size, 2
    return opt


def test_personalize_from_a_frame_equals_from_its_file(cuda, world):
    for on_device in (False, True):
        hmr_p, hmr_f = RecordingHMR(world["v"]), RecordingHMR(world["v"])
        a = Imitator(_opt(), generator=world["net"], hmr=hmr_p, render=_render(world, C.SIZE), device=cuda)
        b = Imitator(_opt(), generator=world["net"], hmr=hmr_f, render=_render(world, C.SIZE), device=cuda)
        out_p, out_f = str(world["root"] / "src_path.png"), str(world["root"] / "src_frame.png")
        a.personalize(world["paths"][0], output_path=out_p)
        frame = torch.from_numpy(world["frames"][0]).to(cuda) if on_device else world["frames"][0]
        b.personalize('', output_path=out_f, src_frame=frame)
        assert torch.equal(a.src_info["img"], b.src_info["img"])
        assert len(hmr_f.inputs) == 1 and torch.equal(hmr_p.inputs[0], hmr_f.inputs[0])
        assert b.src_info["image"] is frame
        for k in ("cond", "bg", "src_inputs"):
            assert torch.equal(a.src_info[k], b.src_info[k]), k
        assert open(out_p, "rb").read() == open(out_f, "rb").read()


@pytest.mark.parametrize("where", ["host", "device", "list"])
def test_inference_from_frames_equals_from_files(cuda, world, where, tmp_path):
    size = 256
    src = S.synthetic_source(size)
    src_theta = np.zeros(85, np.float32)
    src_theta[0] = 0.95

    def make():
        hmr = RecordingHMR(world["v"])
        im = Imitator(_opt(size), generator=world["net"], hmr=hmr, render=_render(world, size), device=cuda)
        im.personalize("", src_smpl=src_theta, src_img=src)
        return im, hmr

    outs = []
    for run in range(2):                                                      # two runs of the file route
        im, hmr_p = make()
        d = tmp_path / ("paths%d" % run)
        d.mkdir()
        outs.append(im.inference(world["paths"], tgt_smpls=None, output_dir=str(d)))
    frames = world["frames"]
    src_frames = {"host": frames, "device": torch.from_numpy(frames).to(cuda), "list": list(frames)}[where]
    im_f, hmr_f = make()
    d_f = tmp_path / "frames"
    d_f.mkdir()
    got = im_f.inference([], tgt_smpls=None, output_dir=str(d_f), tgt_frames=src_frames)

    assert len(hmr_f.inputs) == len(hmr_p.inputs) == 3                       # chunks of 2, 2, 1
    for x, y in zip(hmr_p.inputs, hmr_f.inputs):
        assert torch.equal(x, y)
    for i, p in enumerate(world["paths"]):
        gt_p = cv2.imread(str(tmp_path / "paths0" / ("gt_" + os.path.basename(p))), -1)       # PNG: exact bytes
        gt_f = open(str(d_f / ("gt_%.8d.jpg" % i)), "rb").read()
        assert gt_f == cv2.imencode(".jpg", gt_p)[1].tobytes()                 # the same image through the same encoder
        assert os.path.exists(str(d_f / ("pred_%.8d.jpg" % i)))
    between_runs = max(np.abs(a - b).max() for a, b in zip(outs[0], outs[1]))
    vs_frames = max(np.abs(a - b).max() for a, b in zip(outs[0], got))
    print("inference(tgt_frames, %s) vs paths: max-abs %.3e (two path runs: %.3e)" % (where, vs_frames, between_runs))
    assert vs_frames <= between_runs
    last = im_f.tsf_info["image"]
    assert np.array_equal(last.cpu().numpy() if torch.is_tensor(last) else last, frames[-1])


def test_inference_frames_with_given_smpls_and_argument_conflicts(cuda, world):
    size = C.SIZE
    im = Imitator(_opt(size), generator=world["net"], hmr=RecordingHMR(world["v"]), render=_render(world, size), device=cuda)
    im.personalize('', src_frame=world["frames"][0])
    tgt = np.zeros((3, 85), np.float32)
    tgt[:, 0], tgt[:, 3] = 0.9, [0, 1, 2]
    by_smpls = im.inference_by_smpls(list(tgt))
    with_frames = im.inference([''] * 3, tgt_smpls=list(tgt), tgt_frames=world["frames"][:3])
    assert all(np.array_equal(a, b) for a, b in zip(by_smpls, with_frames))
    with pytest.raises(LwbError, match="both name"):
        im.inference(world["paths"][:3], tgt_frames=world["frames"][:3])
    with pytest.raises(LwbError, match="both name"):
        im.inference([''] * 2, tgt_frames=world["frames"][:3])
    with pytest.raises(LwbError, match="one size"):
        im.inference([], tgt_frames=[world["frames"][0], world["frames"][0][:100]])


def test_inference_over_files_of_two_sizes(cuda, world, tmp_path):
    """Files of two sizes: a chunk whose files share a size is one frames_in launch, a mixed chunk one per file.  Every
    HMR input and every gt_ file is the cv2 route's, bit for bit."""
    size = C.SIZE
    frames = [world["frames"][0], world["frames"][1], world["frames"][2], F.frames(1, 120, 90, seed=12)[0]]
    paths = []
    for i, fr in enumerate(frames):                       # chunks of 2: (333x517, 333x517), (333x517, 120x90)
        paths.append(str(tmp_path / ("t%d.png" % i)))
        cv2.imwrite(paths[-1], fr)
    out = tmp_path / "out"
    out.mkdir()
    hmr = RecordingHMR(world["v"])
    im = Imitator(_opt(size), generator=world["net"], hmr=hmr, render=_render(world, size), device=cuda)
    src_theta = np.zeros(85, np.float32)
    src_theta[0] = 0.95
    im.personalize(world["paths"][0], src_smpl=src_theta)
    got = im.inference(paths, tgt_smpls=None, output_dir=str(out))
    assert len(got) == 4 and len(hmr.inputs) == 2
    hmr_in = torch.cat(hmr.inputs)
    for i, fr in enumerate(frames):
        _, r_hmr, r_gt = F.cv2_route(fr, size)
        assert np.array_equal(_bits(hmr_in[i]), _bits(r_hmr)), i
        ref = str(tmp_path / ("ref%d.png" % i))
        cv2.imwrite(ref, r_gt)
        assert open(str(out / ("gt_t%d.png" % i)), "rb").read() == open(ref, "rb").read(), i
        assert os.path.exists(str(out / ("pred_t%d.png" % i)))
    assert np.array_equal(im.tsf_info["image"], cv2.cvtColor(frames[-1], cv2.COLOR_BGR2RGB))


def test_inference_with_given_smpls_reads_only_the_last_file(cuda, world, monkeypatch):
    """Given SMPL vectors and no output_dir (evaluate.py's call): no file is decoded but the last one, for
    tsf_info['image'], and the frames are those of inference_by_smpls."""
    im = Imitator(_opt(), generator=world["net"], hmr=RecordingHMR(world["v"]), render=_render(world, C.SIZE), device=cuda)
    im.personalize('', src_frame=world["frames"][0])
    tgt = np.zeros((5, 85), np.float32)
    tgt[:, 0], tgt[:, 3] = 0.9, [0, 1, 2, 3, 0]
    reads, imread = [], cv2.imread
    monkeypatch.setattr(cv2, "imread", lambda path, *a: reads.append(path) or imread(path, *a))
    got = im.inference(world["paths"], tgt_smpls=list(tgt))
    assert reads == [world["paths"][-1]]
    assert np.array_equal(im.tsf_info["image"], cv2.cvtColor(world["frames"][-1], cv2.COLOR_BGR2RGB))
    assert all(np.array_equal(a, b) for a, b in zip(got, im.inference_by_smpls(list(tgt))))


def test_viewer_from_a_frame_equals_from_its_file(cuda, world):
    views = []
    for kind in ("path", "frame"):
        vw = Viewer(_opt(), generator=world["net"], hmr=RecordingHMR(world["v"]), render=_render(world, C.SIZE),
                    device=cuda)
        if kind == "path":
            vw.personalize(world["paths"][1])
        else:
            vw.personalize('', src_frame=world["frames"][1])
        views.append(vw.view(np.array([[0, np.pi / 6, 0], [0, -np.pi / 3, 0]], np.float32), [0, 0, 0]).clone())
    assert torch.equal(views[0], views[1])


def test_swapper_from_frames_equals_from_files(cuda, world):
    part_info, _, _ = C.part_table(world["f"].shape[0])
    preds, hmrs = [], []
    for kind in ("path", "frame"):
        hmr = RecordingHMR(world["v"])
        sw = Swapper(_opt(), part_info=part_info, generator=world["net"], hmr=hmr, render=_render(world, C.SIZE),
                     device=cuda)
        if kind == "path":
            sw.swap_setup(world["paths"][2], world["paths"][3])
        else:
            sw.swap_setup('', '', src_frame=world["frames"][2], tgt_frame=torch.from_numpy(world["frames"][3]).to(cuda))
        hmrs.append(hmr.inputs)
        preds.append(sw.swap(sw.src_info, sw.tsf_info, target_part="body").clone())
        if kind == "path":
            ref_imgs = (sw.src_info["img"], sw.tsf_info["img"])
        else:
            assert torch.equal(ref_imgs[0], sw.src_info["img"]) and torch.equal(ref_imgs[1], sw.tsf_info["img"])
    assert len(hmrs[1]) == 2 and all(torch.equal(x, y) for x, y in zip(hmrs[0], hmrs[1]))
    assert torch.equal(preds[0], preds[1])
