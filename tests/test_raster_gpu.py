"""GPU parity of the rasterizer / correspondence kernels (through the C ABI) against
  * the reference's own CUDA kernels (bit-exact: SHA-256 digests of their outputs on the same inputs, recorded on an H100
    by tests/golden/make_raster_golden.py, are stored in tests/golden/raster_ref_kernels.json), and
  * the C restatement (oracle/raster_ref.c) + torch glue restatement (oracle/nmr_ref.py)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

from impersonator_b200 import kernels as K
from impersonator_b200 import synthetic as S
from oracle import nmr_ref, raster

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
# the tests whose inputs are compared with the reference kernels (tests/golden/make_raster_golden.py replays them)
REFERENCE_COMPARED = ("test_sphere_bit_exact_vs_reference_kernels", "test_sphere_512_bit_exact",
                      "test_teapot_batch_with_degenerate_meshes", "test_random_triangle_soup_bit_exact",
                      "test_big_faces_bit_exact_and_grid_wide")


def run_mine(faces, size, flip=False, want_inv=True):
    B, F = faces.shape[:2]
    dev = faces.device
    fim = torch.full((B, size, size), -1, dtype=torch.int32, device=dev)
    wim = torch.zeros((B, size, size, 3), dtype=torch.float32, device=dev)
    depth = torch.full((B, size, size), 100.0, dtype=torch.float32, device=dev)
    finv = torch.zeros((B, F, 3, 3), dtype=torch.float32, device=dev) if want_inv else None
    K.raster_forward_face_index_map(faces, fim, wim, depth, size, faces_inv=finv, flip_rows=flip)
    torch.cuda.synchronize()
    return fim, wim, depth, finv


def digests(fim, wim, depth, finv):
    d = lambda t: hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()
    return {"faces_inv": d(finv), "fim": d(fim), "wim": d(wim), "depth": d(depth), "covered": int((fim >= 0).sum())}


def compare_with_gpu_ref(faces, size, key):
    """Outputs bit for bit equal to the reference kernels' outputs for the same input (stored digests, see module doc)."""
    fim, wim, depth, finv = run_mine(faces, size)
    with open(os.path.join(GOLD, "raster_ref_kernels.json")) as f:
        want = json.load(f)[key]
    got = digests(fim, wim, depth, finv)
    print("%s: covered %d (reference %d)" % (key, got["covered"], want["covered"]))
    assert got["faces_inv"] == want["faces_inv"], "faces_inv differs bitwise from the reference kernel_1"
    assert got["fim"] == want["fim"], "face_index_map differs from the reference kernel_2"
    assert got["wim"] == want["wim"] and got["depth"] == want["depth"]
    return fim


def sphere_faces(B, seed, dev):
    v, f = S.uv_sphere()
    cam, verts = S.synthetic_frames(B, seed=seed, base_verts=v)
    return nmr_ref.project_to_faces(cam, verts, f).to(dev).contiguous(), cam, verts, f


def test_sphere_bit_exact_vs_reference_kernels(cuda):
    faces, _, _, _ = sphere_faces(3, 1234, cuda)
    for size in (256, 64):
        fim = compare_with_gpu_ref(faces, size, "sphere3/1234/%d" % size)
        assert int((fim >= 0).sum()) > 100


def test_sphere_512_bit_exact(cuda):
    faces, _, _, _ = sphere_faces(2, 77, cuda)
    compare_with_gpu_ref(faces, 512, "sphere2/77/512")


def test_teapot_batch_with_degenerate_meshes(cuda):
    """tests/utils.py:11-27 (to_minibatch): the teapot sits in slot 2 of a batch of 4, the other
    three meshes are all-zero vertices -> every face degenerate (whole-image scan path)."""
    g = np.load(os.path.join(GOLD, "teapot.npz"))
    tp = torch.from_numpy(g["faces"])
    zero_v = torch.zeros(1, 1292, 3)
    # the all-zero mesh after look_at + perspective (look_at.py:57-60, perspective.py:13-20)
    z = zero_v[..., 2] - nmr_ref.EYE_Z
    width = torch.tan(torch.tensor(30. / 180 * np.pi))
    zv = torch.stack((zero_v[..., 0] / z / width, zero_v[..., 1] / z / width, z), dim=2)
    zf = zv[0][torch.zeros(tp.shape[0], 3, dtype=torch.long)]
    faces = torch.stack([zf, zf, tp, zf]).to(cuda).contiguous()
    fim = compare_with_gpu_ref(faces, 256, "teapot/256")
    sil = np.unpackbits(g["silhouette"]).reshape(256, 256).astype(bool)
    mine = (fim[2].flip(0) >= 0).cpu().numpy()
    assert (mine != sil).sum() == 0                      # test_rasterize_silhouettes.py:16-35
    assert int((fim[[0, 1, 3]] >= 0).sum()) == 0


def random_soup(B, F, seed):
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(B, F, 1, 2, generator=g) * 2.4 - 1.2
    size = torch.rand(B, F, 1, 1, generator=g) ** 3 * 0.8 + 0.002
    xy = c + (torch.rand(B, F, 3, 2, generator=g) - 0.5) * size
    z = 1.0 + torch.rand(B, F, 3, 1, generator=g) * 3
    faces = torch.cat([xy, z], dim=-1)
    faces[:, 1::7] = faces[:, 0::7][:, :faces[:, 1::7].shape[1]]          # exact duplicates -> depth ties
    faces[:, 5::11, :, 2] = 2.0                                           # coplanar constant depth -> many ties
    faces[:, 3::50, 1] = faces[:, 3::50, 0]                               # two identical vertices (zero area)
    faces[:, 4::53] = faces[:, 4::53, :1]                                 # all three identical
    faces[:, 9::61, :, 0] = faces[:, 9::61, :1, 0]                        # vertical collinear
    faces[0, 7::97, 0, 2] = 0.05                                          # vertices nearer than `near`
    faces[0, 8::89, :, :2] *= 30                                          # huge triangles
    return faces.float().contiguous()


def test_random_triangle_soup_bit_exact(cuda):
    for seed, size in ((1, 128), (2, 256), (3, 96)):
        compare_with_gpu_ref(random_soup(2, 3000, seed).to(cuda), size, "soup/%d/%d" % (seed, size))


def test_big_faces_bit_exact_and_grid_wide(cuda):
    """Many faces covering thousands of pixels each (boxes > kBigBox go to the grid-wide scan instead of one warp): bit-exact
    against the reference kernels, and not a straggler."""
    g = torch.Generator().manual_seed(11)
    B, F = 2, 1500
    c = torch.rand(B, F, 1, 2, generator=g) * 1.6 - 0.8
    size = 0.2 + torch.rand(B, F, 1, 1, generator=g) * 1.2                 # 25..180 px wide at 256^2
    xy = c + (torch.rand(B, F, 3, 2, generator=g) - 0.5) * size
    z = 1.0 + torch.rand(B, F, 3, 1, generator=g) * 3
    faces = torch.cat([xy, z], dim=-1).float().contiguous().to(cuda)
    compare_with_gpu_ref(faces, 256, "big_faces/256")
    for _ in range(3):
        run_mine(faces, 256, want_inv=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        run_mine(faces, 256, want_inv=False)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    print("3000 large faces (avg box ~10^4 px) @256^2: %.3f ms" % ms)
    assert ms < 5.0


def test_flip_rows_matches_torch_flip(cuda):
    faces, _, _, _ = sphere_faces(2, 5, cuda)
    a = run_mine(faces, 256, flip=False, want_inv=False)
    b = run_mine(faces, 256, flip=True, want_inv=False)
    assert torch.equal(a[0].flip(1), b[0]) and torch.equal(a[1].flip(1), b[1]) and torch.equal(a[2].flip(1), b[2])


def test_raster_matches_c_oracle(cuda):
    faces, _, _, _ = sphere_faces(2, 99, cuda)
    fim, wim, depth, finv = run_mine(faces, 256)
    ofim, owim, odepth, ofinv = raster.forward_face_index_map_cpu(faces.cpu().numpy(), 256)
    assert int((fim.cpu().numpy() != ofim).sum()) == 0
    assert np.array_equal(finv.cpu().numpy().view(np.int32), ofinv.view(np.int32))
    assert np.abs(wim.cpu().numpy() - owim).max() == 0
    assert np.abs(depth.cpu().numpy() - odepth).max() == 0


@pytest.mark.parametrize("align_corners", [False, True])
def test_correspond_matches_oracle(cuda, align_corners):
    """lwb_correspond vs the restated torch glue (models/imitator.py:251-260)."""
    v, f = S.uv_sphere()
    cam, verts = S.synthetic_frames(3, seed=42, base_verts=v)
    tabs = S.synthetic_tables()
    src_img = S.synthetic_source(256)
    f2v_src, _, _ = nmr_ref.render_fim_wim(cam[:1], verts[:1], f, 256)
    p2v = nmr_ref.src_p2verts(f2v_src)
    ref = nmr_ref.correspond(cam[1:], verts[1:], f, tabs["map_fn"], p2v, src_img, 256, align_corners)
    out = K.correspond(cam[1:].to(cuda).contiguous(), verts[1:].to(cuda).contiguous(), f.to(cuda), 256,
                       tabs["map_fn"].to(cuda), p2v.to(cuda).contiguous(), src_img.to(cuda),
                       align_corners=align_corners, want_f2verts=True)
    torch.cuda.synchronize()
    assert torch.equal(out["f2verts"].cpu(), ref["f2verts"])
    assert int((out["fim"].cpu() != ref["fim"]).sum()) == 0
    for k, tol in (("wim", 1e-6), ("T", 1e-5), ("cond", 0.0), ("tsf_img", 2e-5), ("tsf_inputs", 2e-5)):
        d = (out[k].cpu() - ref[k]).abs().max().item()
        print(k, d)
        assert d <= tol, (k, d)


def test_correspond_source_pass_matches_render_fim_wim(cuda):
    """personalize-side use (models/imitator.py:100-107): f2verts / fim / wim only."""
    v, f = S.uv_sphere()
    cam, verts = S.synthetic_frames(1, seed=8, base_verts=v)
    tabs = S.synthetic_tables()
    f2v, fim, wim = nmr_ref.render_fim_wim(cam, verts, f, 256)
    p2v = nmr_ref.src_p2verts(f2v)
    out = K.correspond(cam.to(cuda), verts.to(cuda), f.to(cuda), 256, tabs["map_fn"].to(cuda), p2v.to(cuda).contiguous(),
                       None, want_f2verts=True)
    assert torch.equal(out["fim"].cpu(), fim)
    assert (out["wim"].cpu() - wim).abs().max().item() <= 1e-6
    # self-correspondence: T of the source onto itself reproduces pixel centres (sanity of cal_bc_transform)
    T = out["T"].cpu()
    cov = fim[0] >= 0
    ys, xs = torch.meshgrid(torch.arange(256), torch.arange(256), indexing="ij")
    gx = (2.0 * xs + 1 - 256) / 256
    assert (T[0][cov][:, 0] - gx[cov]).abs().max().item() < 2e-2


def test_self_correspondence_is_the_identity_warp(cuda):
    """Round trip through lwb_correspond at the full 256^2 / 512^2 sizes: frame 0 corresponded with itself gives
    T = pixel centres and tsf_img = src_img on covered pixels, -2 / 0 elsewhere (no oracle involved).  The image identity
    holds in the align_corners=False sampling convention (pixel centres are the rasterizer's sample points); the default
    torch-1.2 convention shifts the sample by <= half a pixel, exactly as the reference did."""
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    for size in (256, 512):
        cam, verts = S.synthetic_frames(2, seed=8, base_verts=v)
        ys, xs = torch.meshgrid(torch.arange(size, dtype=torch.float32), torch.arange(size, dtype=torch.float32), indexing="ij")
        gx, gy = (2 * xs + 1 - size) / size, (2 * ys + 1 - size) / size
        src = torch.stack([torch.sin(3 * gx) * torch.cos(2 * gy), gx * gy, torch.cos(4 * gx + gy)])[None]
        from impersonator_b200.nmr import SMPLRenderer
        r = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"]).to(cuda)
        src_pass = r.correspond(cam[:1].to(cuda), verts[:1].to(cuda), None, None, want_f2verts=True)     # personalize side
        p2v = src_pass["f2verts"][:, :, :, 0:2].clone()
        p2v[:, :, :, 1] *= -1                                                  # models/imitator.py:105-107
        out = r.correspond(cam.to(cuda), verts.to(cuda), p2v.contiguous(), src.to(cuda), align_corners=False)
        torch.cuda.synchronize()
        fim, T, img = out["fim"][0].cpu(), out["T"][0].cpu(), out["tsf_img"][0].cpu()
        cov = fim >= 0
        assert 0.05 < cov.float().mean() < 0.6
        # a quarter of a pixel at most (worst on sliver faces, where the reference's clamped barycentrics are least exact)
        assert (T[..., 0] - gx)[cov].abs().max() < 0.5 / size and (T[..., 1] - gy)[cov].abs().max() < 0.5 / size
        assert (T[..., 0] - gx)[cov].abs().mean() < 2e-5
        assert torch.all(T[~cov] == -2) and torch.all(img[:, ~cov] == 0)
        assert (img - src[0])[:, cov].abs().max() < 5e-3


def _correspond_args(cuda, B=2, s=16, F=4, V=5, C=3, sb=1):
    return dict(cam=torch.ones(B, 3, device=cuda), verts=torch.zeros(B, V, 3, device=cuda),
                face_idx=torch.zeros(F, 3, dtype=torch.int32, device=cuda), image_size=s,
                map_fn=torch.zeros(F + 1, C, device=cuda), src_p2verts=torch.zeros(sb, F, 3, 2, device=cuda),
                src_img=torch.zeros(sb, 3, s, s, device=cuda))


def _correspond_out(cuda, B=2, s=16, F=4, C=3):
    return dict(fim=torch.zeros(B, s, s, dtype=torch.int32, device=cuda), wim=torch.zeros(B, s, s, 3, device=cuda),
                T=torch.zeros(B, s, s, 2, device=cuda), tsf_inputs=torch.zeros(B, 3 + C, s, s, device=cuda),
                f2verts=torch.zeros(B, F, 3, 3, device=cuda))


CORRESPOND_BAD = {
    "cam [B,2]": lambda a, o, c: a.update(cam=torch.ones(2, 2, device=c)),
    "cam of another batch": lambda a, o, c: a.update(cam=torch.ones(3, 3, device=c)),
    "cam float64": lambda a, o, c: a.update(cam=torch.ones(2, 3, dtype=torch.float64, device=c)),
    "verts [B,V,2]": lambda a, o, c: a.update(verts=torch.zeros(2, 5, 2, device=c)),
    "face_idx [F,4]": lambda a, o, c: a.update(face_idx=torch.zeros(4, 4, dtype=torch.int32, device=c)),
    "face_idx int64": lambda a, o, c: a.update(face_idx=torch.zeros(4, 3, dtype=torch.int64, device=c)),
    "map_fn rows": lambda a, o, c: a.update(map_fn=torch.zeros(4, 3, device=c)),
    "src_p2verts batch 3 of 2": lambda a, o, c: a.update(src_p2verts=torch.zeros(3, 4, 3, 2, device=c),
                                                         src_img=torch.zeros(3, 3, 16, 16, device=c)),
    "src_p2verts faces": lambda a, o, c: a.update(src_p2verts=torch.zeros(1, 5, 3, 2, device=c)),
    "src_p2verts [sb,F,3,3]": lambda a, o, c: a.update(src_p2verts=torch.zeros(1, 4, 3, 3, device=c)),
    "src_img of another size": lambda a, o, c: a.update(src_img=torch.zeros(1, 3, 32, 32, device=c)),
    "src_img batch B, src_p2verts batch 1": lambda a, o, c: a.update(src_img=torch.zeros(2, 3, 16, 16, device=c)),
    "src_img 4 channels": lambda a, o, c: a.update(src_img=torch.zeros(1, 4, 16, 16, device=c)),
    "out fim shape": lambda a, o, c: o.update(fim=torch.zeros(2, 16, 15, dtype=torch.int32, device=c)),
    "out fim float32": lambda a, o, c: o.update(fim=torch.zeros(2, 16, 16, device=c)),
    "out wim shape": lambda a, o, c: o.update(wim=torch.zeros(2, 16, 16, 2, device=c)),
    "out T shape": lambda a, o, c: o.update(T=torch.zeros(1, 16, 16, 2, device=c)),
    "out tsf_inputs channels": lambda a, o, c: o.update(tsf_inputs=torch.zeros(2, 3, 16, 16, device=c)),
    "out f2verts faces": lambda a, o, c: o.update(f2verts=torch.zeros(2, 3, 3, 3, device=c)),
}


@pytest.mark.parametrize("bad", sorted(CORRESPOND_BAD))
def test_correspond_rejects_mismatched_shapes(cuda, bad):
    """Every input and caller buffer is checked against the shapes the kernel indexes with (B, F, sb, image size): a
    source image of another size or batch, or a short buffer, is an LwbError, not an out-of-bounds read or write."""
    a, o = _correspond_args(cuda), _correspond_out(cuda)
    CORRESPOND_BAD[bad](a, o, cuda)
    with pytest.raises(K.LwbError):
        K.correspond(a.pop("cam"), a.pop("verts"), a.pop("face_idx"), a.pop("image_size"), a.pop("map_fn"),
                     a.pop("src_p2verts"), a.pop("src_img"), want_f2verts=True, out=o)


RASTER_BAD = ["faces [B,F,3,2]", "faces [B,F,9]", "faces float64", "fim shape", "fim int64", "wim shape", "depth shape",
              "faces_inv faces"]


@pytest.mark.parametrize("bad", RASTER_BAD)
def test_raster_forward_rejects_mismatched_shapes(cuda, bad):
    B, F, s = 2, 4, 16
    faces = torch.zeros(B, F, 3, 3, device=cuda)
    fim = torch.full((B, s, s), -1, dtype=torch.int32, device=cuda)
    wim = torch.zeros(B, s, s, 3, device=cuda)
    depth = torch.zeros(B, s, s, device=cuda)
    finv = torch.zeros(B, F, 3, 3, device=cuda)
    if bad == "faces [B,F,3,2]":
        faces = torch.zeros(B, F, 3, 2, device=cuda)
    elif bad == "faces [B,F,9]":
        faces = torch.zeros(B, F, 9, device=cuda)
    elif bad == "faces float64":
        faces = torch.zeros(B, F, 3, 3, dtype=torch.float64, device=cuda)
    elif bad == "fim shape":
        fim = torch.full((B, s, s + 1), -1, dtype=torch.int32, device=cuda)
    elif bad == "fim int64":
        fim = torch.full((B, s, s), -1, dtype=torch.int64, device=cuda)
    elif bad == "wim shape":
        wim = torch.zeros(B, s, s, device=cuda)
    elif bad == "depth shape":
        depth = torch.zeros(1, s, s, device=cuda)
    else:
        finv = torch.zeros(B, F + 1, 3, 3, device=cuda)
    with pytest.raises(K.LwbError):
        K.raster_forward_face_index_map(faces, fim, wim, depth, s, faces_inv=finv)
