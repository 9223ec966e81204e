"""Synthetic stand-ins for the assets the reference downloads (SURVEY.md section 0 fact 5, section 8d).

Nothing the hot path needs at run time ships with the reference (``assets/pretrains/*`` and
``outputs/checkpoints/*`` are external downloads, README.md:48-68), so tests, ``bench.py`` and
``smoke()`` drive the path with:

* a UV-sphere with 84 rings x 82 segments + 2 poles: V = 6890, F = 13776 = 2V - 4, exactly the
  SMPL counts (utils/nmr.py:620, networks/batch_smpl.py:252), consistently wound so that the
  reference's back-face test (rasterize_cuda_kernel.cu:57) keeps the camera-facing half;
* per-frame "poses" = rigid rotations + a smooth vertex displacement, weak-perspective cams
  ``[s, tx, ty]`` as HMR emits them (utils/nmr.py:10-28);
* lookup tables shaped like utils/mesh.py:368-421 (``map_fn`` (F+1) x 3 with background row
  ``[0, 0, 1]``, front/back masks (F+1) x 1);
* deterministic, key-addressed random weights with the reference's ``state_dict`` keys and
  shapes (N(0, 0.02) convs as networks/networks.py:54-65, non-trivial norm affines).

Everything is seeded and device independent (generated on CPU with torch.Generator).
"""
import hashlib
import math

import numpy as np
import torch

SMPL_V = 6890
SMPL_F = 13776


def uv_sphere(rings=84, segments=82, radii=(0.35, 0.9, 0.25)):
    """-> (verts f32[V,3], faces i32[F,3]) with V = rings*segments + 2, F = 2*rings*segments.

    Winding is chosen so that, after the renderer's y-flip and z-offset (utils/nmr.py:271-273),
    triangles on the camera side (z < 0 before the offset, i.e. nearer the eye at z = -2.73)
    pass ``(y2-y0)*(x1-x0) >= (y1-y0)*(x2-x0)``.
    """
    verts = []
    for r in range(rings):
        theta = math.pi * (r + 1) / (rings + 1)
        for s in range(segments):
            phi = 2 * math.pi * s / segments
            verts.append((math.sin(theta) * math.cos(phi), math.cos(theta), math.sin(theta) * math.sin(phi)))
    north = len(verts)
    verts.append((0.0, 1.0, 0.0))
    south = len(verts)
    verts.append((0.0, -1.0, 0.0))
    faces = []
    for s in range(segments):
        s1 = (s + 1) % segments
        faces.append((north, s1, s))
        base = (rings - 1) * segments
        faces.append((south, base + s, base + s1))
    for r in range(rings - 1):
        for s in range(segments):
            s1 = (s + 1) % segments
            a, b = r * segments + s, r * segments + s1
            c, d = (r + 1) * segments + s, (r + 1) * segments + s1
            faces.append((a, b, c))
            faces.append((b, d, c))
    verts = np.asarray(verts, np.float32) * np.asarray(radii, np.float32)[None]
    faces = np.asarray(faces, np.int32)
    return torch.from_numpy(verts), torch.from_numpy(faces)


def _rot(ax, ang):
    c, s = math.cos(ang), math.sin(ang)
    if ax == 'y':
        return torch.tensor([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=torch.float32)
    return torch.tensor([[1, 0, 0], [0, c, -s], [0, s, c]], dtype=torch.float32)


def synthetic_frames(batch, seed=1234, base_verts=None):
    """-> cam f32[B,3], verts f32[B,V,3]: rotation about y ~U(-pi,pi), about x ~U(-0.3,0.3),
    smooth displacement, cam = [s~U(0.8,1.1), tx,ty~U(-0.1,0.1)] (SURVEY.md 8d)."""
    g = torch.Generator().manual_seed(seed)
    if base_verts is None:
        base_verts, _ = uv_sphere()
    out_v, out_c = [], []
    for _ in range(batch):
        u = torch.rand(8, generator=g)
        ry = (u[0].item() * 2 - 1) * math.pi
        rx = (u[1].item() * 2 - 1) * 0.3
        v = base_verts @ _rot('y', ry).T @ _rot('x', rx).T
        k = 2 + 3 * u[2].item()
        amp = 0.02 + 0.02 * u[3].item()
        v = v + amp * torch.stack([torch.sin(k * v[:, 1] + u[4] * 6), torch.cos(k * v[:, 0] + u[5] * 6),
                                   torch.sin(k * v[:, 0] * 0.5)], dim=1)
        out_v.append(v.float())
        out_c.append(torch.tensor([0.8 + 0.3 * u[6].item(), (u[7].item() * 2 - 1) * 0.1,
                                   (torch.rand(1, generator=g).item() * 2 - 1) * 0.1], dtype=torch.float32))
    return torch.stack(out_c), torch.stack(out_v)


def synthetic_tables(num_faces=SMPL_F, seed=7):
    """-> dict(map_fn f32[F+1,3], front_map_fn f32[F+1,1], back_map_fn f32[F+1,1])
    shaped like utils/mesh.py:368-421 ('uv_seg' :399-402; background row :418-419)."""
    g = torch.Generator().manual_seed(seed)
    map_fn = torch.zeros(num_faces + 1, 3)
    map_fn[:num_faces, :2] = torch.rand(num_faces, 2, generator=g)
    map_fn[num_faces] = torch.tensor([0.0, 0.0, 1.0])
    front = (torch.rand(num_faces + 1, 1, generator=g) < 0.05).float()
    back = (torch.rand(num_faces + 1, 1, generator=g) < 0.05).float()
    front[num_faces] = 0
    back[num_faces] = 0
    return dict(map_fn=map_fn, front_map_fn=front, back_map_fn=back)


def _key_gen(seed, key):
    h = hashlib.sha256(("%d/%s" % (seed, key)).encode()).digest()
    return torch.Generator().manual_seed(int.from_bytes(h[:7], 'little'))


def fill_state_dict(template, seed=0, conv_std=0.02):
    """Deterministic weights for a ``state_dict``-shaped template (key -> tensor or shape).

    Values depend only on (seed, key, shape): >=2-D tensors ~ N(0, conv_std) (``conv_std='he'``: N(0, 2 / fan_in),
    which keeps activations O(1) through BatchNorm-in-eval networks such as the HMR encoder); 1-D ``*.weight``
    ~ 1 + 0.1 N(0,1) (norm scales); 1-D ``*.bias`` ~ 0.1 N(0,1); ``running_var`` ~ U(0.5, 1.5);
    ``running_mean`` ~ 0.1 N(0,1); integer buffers (``num_batches_tracked``) = 0.
    """
    out = {}
    for key, t in template.items():
        shape = tuple(t.shape) if hasattr(t, 'shape') else tuple(t)
        dtype = t.dtype if hasattr(t, 'dtype') else torch.float32
        g = _key_gen(seed, key)
        if not dtype.is_floating_point:
            out[key] = torch.zeros(shape, dtype=dtype)
        elif len(shape) >= 2:
            std = conv_std
            if conv_std == 'he':
                fan_in = 1
                for d in shape[1:]:
                    fan_in *= d
                std = math.sqrt(2.0 / fan_in)
            out[key] = torch.randn(shape, generator=g) * std
        elif key.endswith('running_var'):
            out[key] = 0.5 + torch.rand(shape, generator=g)
        elif key.endswith('running_mean'):
            out[key] = 0.1 * torch.randn(shape, generator=g)
        elif key.endswith('gamma'):
            out[key] = 0.5 + 0.0 * torch.randn(shape, generator=g)
        elif key.endswith('weight'):
            out[key] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        else:
            out[key] = 0.1 * torch.randn(shape, generator=g)
    return out


def synthetic_source(image_size=256, seed=99):
    """-> src_img f32[1,3,H,W] in [-1,1] (smooth, so bilinear warps are well conditioned)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(1, 3, image_size // 8, image_size // 8, generator=g) * 2 - 1
    img = torch.nn.functional.interpolate(low, size=(image_size, image_size), mode='bilinear', align_corners=False)
    return (img + 0.1 * (torch.rand(1, 3, image_size, image_size, generator=g) - 0.5)).clamp(-1, 1)


def synthetic_flow(batch, image_size=256, seed=5):
    """-> T f32[B,H,W,2]: smooth flow in about [-1.1, 1.1] inside an ellipse, -2 outside
    (the background value cal_bc_transform writes, utils/nmr.py:627)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(batch, 2, 6, 6, generator=g) * 2.2 - 1.1
    T = torch.nn.functional.interpolate(low, size=(image_size, image_size), mode='bicubic', align_corners=True)
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, image_size), torch.linspace(-1, 1, image_size), indexing='ij')
    inside = ((xs / 0.55) ** 2 + (ys / 0.9) ** 2) < 1
    T = T.permute(0, 2, 3, 1).contiguous()
    T[:, ~inside] = -2.0
    return T


def synthetic_generator_inputs(batch, image_size=256, seed=11):
    """-> dict(bg f32[1,4,H,W], src f32[1,6,H,W], tsf f32[B,6,H,W], T f32[B,H,W,2]) in [-1,1]."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g) * 2 - 1
    return dict(bg=r(1, 4, image_size, image_size), src=r(1, 6, image_size, image_size),
                tsf=r(batch, 6, image_size, image_size), T=synthetic_flow(batch, image_size, seed + 1))


# SMPL kinematic tree (kintree_table[0] of the public SMPL model; entry 0 is the root, stored as uint32 -1)
SMPL_PARENTS = (-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21)


def synthetic_smpl_model(seed=3, num_betas=10, num_joints=19):
    """A stand-in for ``smpl_model.pkl`` (external, not redistributable) with the SAME keys, shapes and
    dtypes that ``SMPL.__init__`` reads (networks/batch_smpl.py:236-283): the UV-sphere body as template,
    random blend shapes, banded joint regressors and 4-joint skinning weights.  numpy / scipy.sparse only."""
    import scipy.sparse as sp
    rs = np.random.RandomState(seed)
    v, f = uv_sphere()
    v = v.numpy().astype(np.float64)
    V = v.shape[0]
    order = np.argsort(v[:, 1], kind="stable")                 # bottom to top
    band = np.empty(V, dtype=np.int64)
    band[order] = (np.arange(V) * 24) // V                        # 24 height bands <-> 24 joints

    def banded(rows, per_row):
        m = np.zeros((rows, V), dtype=np.float64)
        for j in range(rows):
            cand = np.nonzero(band == (j * 24) // rows)[0]
            idx = rs.choice(cand, size=per_row, replace=False)
            w = rs.rand(per_row) + 0.1
            m[j, idx] = w / w.sum()
        return sp.csc_matrix(m)

    # smooth skinning weights: a Gaussian over the (continuous) height coordinate, 4 nearest joints kept
    t = np.empty(V, dtype=np.float64)
    t[order] = (np.arange(V) + 0.5) * 24.0 / V - 0.5
    weights = np.exp(-0.5 * ((t[:, None] - np.arange(24)[None, :]) / 0.8) ** 2)
    kth = np.sort(weights, axis=1)[:, -4][:, None]
    weights = np.where(weights >= kth, weights, 0.0)
    weights /= weights.sum(axis=1, keepdims=True)
    # smooth (low-frequency) blend shapes: 12 basis functions of the vertex position, random mixing
    ang = np.arctan2(v[:, 2], v[:, 0])
    basis = np.stack([np.ones(V), v[:, 1], v[:, 1] ** 2, np.sin(3 * v[:, 1]), np.cos(3 * v[:, 1]), np.sin(ang), np.cos(ang),
                      np.sin(2 * ang), np.cos(2 * ang), np.sin(ang) * v[:, 1], np.cos(ang) * v[:, 1], np.sin(6 * v[:, 1])], axis=1)

    def smooth_dirs(n, scale):
        return np.einsum('vi,idk->vdk', basis, rs.randn(basis.shape[1], 3, n)) * scale
    kintree = np.zeros((2, 24), dtype=np.uint32)
    kintree[0] = np.array(SMPL_PARENTS, dtype=np.int64).astype(np.uint32)
    kintree[1] = np.arange(24)
    return {
        "f": f.numpy().astype(np.uint32),
        "v_template": v,
        "shapedirs": smooth_dirs(num_betas, 0.004),
        "posedirs": smooth_dirs(207, 0.0015),
        "J_regressor": banded(24, 40),
        "kintree_table": kintree,
        "weights": weights,
        "cocoplus_regressor": banded(num_joints, 24),
    }


def synthetic_smpl_params(batch, seed=17):
    """-> theta f32[B,85] = [cam(3) | pose(72) | shape(10)] (the layout of networks/hmr.py:314-316)."""
    g = torch.Generator().manual_seed(seed)
    cam = torch.stack([0.8 + 0.3 * torch.rand(batch, generator=g), torch.rand(batch, generator=g) * 0.2 - 0.1,
                       torch.rand(batch, generator=g) * 0.2 - 0.1], dim=1)
    pose = torch.randn(batch, 72, generator=g) * 0.1
    pose[:, 0:3] = torch.stack([torch.randn(batch, generator=g) * 0.2, (torch.rand(batch, generator=g) * 2 - 1) * math.pi,
                                torch.randn(batch, generator=g) * 0.1], dim=1)
    shape = torch.randn(batch, 10, generator=g)
    return torch.cat([cam, pose, shape], dim=1).float()


def synthetic_hmr_inputs(batch, seed=9):
    """-> images f32[B,3,224,224] in [-1,1] as HumanModelRecovery.forward receives them (models/imitator.py:93-95)."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(batch, 3, 28, 28, generator=g) * 2 - 1
    img = torch.nn.functional.interpolate(low, size=(224, 224), mode='bilinear', align_corners=False)
    return (img + 0.2 * (torch.rand(batch, 3, 224, 224, generator=g) - 0.5)).clamp(-1, 1)


def synthetic_hmr_state(template, seed=4):
    """Deterministic ``resnet.*`` / ``regressor.*`` entries for a HumanModelRecovery ``state_dict`` template (the
    released hmr_tf2pt.pth is an external download; 27 M parameters are regenerated from the seed wherever needed).
    He-scaled convs with the last conv of every residual branch damped (16 unit-gain branches would push the
    pre-activation stream to |x| ~ 1e3), mean_theta like load_mean_theta (networks/hmr.py:190-211): scale 0.9, upright."""
    sd = fill_state_dict({k: v for k, v in template.items() if not k.startswith("smpl.")}, seed=seed, conv_std='he')
    mt = torch.zeros(85)
    mt[0], mt[3] = 0.9, math.pi
    mt[75:] = 0.1 * torch.randn(10, generator=torch.Generator().manual_seed(seed))
    sd["regressor.mean_theta"] = mt
    sd["regressor.fc_blocks.fc3.weight"] = sd["regressor.fc_blocks.fc3.weight"] * 0.03    # small_xavier (hmr.py:231)
    for k in sd:
        if sd[k].dim() == 4 and ".conv3." in k:
            sd[k] = sd[k] * 0.25
    return sd


def synthetic_maskrcnn_state(seed=21, person_bias=5.0):
    """Deterministic weights for the Mask R-CNN detector, with the published COCO checkpoint's (version-1) keys (the
    44.5 M parameters are regenerated from the seed wherever they are needed).  He-scaled convs and linears, FrozenBN
    statistics as in fill_state_dict, the last conv of every bottleneck damped (post-add ReLU: 16 unit-gain branches
    would grow the stream ~30x), the RPN and box predictors damped (objectness and class logits of order 1, as a trained model's: saturated
    sigmoids would tie), box and anchor deltas small so boxes stay near their anchors / proposals, and the
    person class's ``cls_score`` bias raised by ``person_bias`` so that several person detections exist."""
    from .detectors import MaskRCNN, to_v1
    template = {k: tuple(v.shape) for k, v in MaskRCNN().state_dict().items()}
    sd = fill_state_dict(template, seed=seed, conv_std='he')
    for k in sd:
        if ".conv3." in k and sd[k].dim() == 4:
            sd[k] = sd[k] * 0.25
        if k.endswith("bbox_pred.weight") or k.endswith("cls_logits.weight") or k.endswith("cls_score.weight"):
            sd[k] = sd[k] * 0.1
    sd["roi_heads.box_predictor.cls_score.bias"][1] += person_bias
    return to_v1(sd)


class QuarterTurnBodyModel(object):
    """A body model whose vertices are EXACT on every device: theta[3] = k selects a rotation of the UV-sphere body by
    k quarter turns about y (a signed permutation of coordinates, no rounding), theta[0:3] = cam.  Used where a CPU-made
    golden and the GPU path must rasterize bit-identical vertices (cos / sin differ by an ulp between devices)."""

    def __init__(self, base_verts):
        self.base = base_verts

    def get_details(self, theta):
        dev = theta.device
        base = self.base.to(dev)
        x, y, z = base[:, 0], base[:, 1], base[:, 2]
        turned = [torch.stack(c, dim=1) for c in ((x, y, z), (z, y, -x), (-x, y, -z), (-z, y, x))]
        ks = [int(round(float(k))) % 4 for k in theta[:, 3].tolist()]
        verts = torch.stack([turned[k] for k in ks], dim=0).contiguous()
        return {'theta': theta, 'cam': theta[:, 0:3].contiguous(), 'pose': theta[:, 3:75].contiguous(),
                'shape': theta[:, 75:].contiguous(), 'verts': verts, 'j2d': None, 'j3d': None}


def save_png(img, path):
    """[3,H,W] float in [-1,1] -> 8-bit BGR png (what cv2.imread gives back to the loaders)."""
    import cv2
    a = ((img.permute(1, 2, 0).numpy() + 1) * 127.5).round().clip(0, 255).astype(np.uint8)
    cv2.imwrite(path, a[..., ::-1].copy())


def synthetic_part_info(n_parts=10):
    """Stand-in for assets/pretrains/smpl_part_info.json (utils/mesh.py:247-268): ``n_parts`` named parts covering every
    face once -- horizontal bands of the UV-sphere body (its faces are ordered ring by ring); part 0 is the top 30 %."""
    head = int(0.3 * SMPL_F)                                      # part 0 (what PART_IDS['body'] leaves alone): a sizeable "head"
    bounds = np.concatenate([[0], np.linspace(head, SMPL_F, n_parts).astype(int)])
    return {"%02d_part" % i: {"face": list(range(int(bounds[i]), int(bounds[i + 1])))} for i in range(n_parts)}


def write_synthetic_assets(root, image_size=256, n_targets=3, seed=0):
    """Everything ``Imitator(opt)`` loads from disk in the reference, as synthetic files with the real formats
    (README.md:48-68 lists the real downloads): under ``root``

      assets/pretrains/smpl_faces.npy       int faces [13776, 3]                       utils/nmr.py:137
      assets/pretrains/mapper.txt           obj-style v / vn / vt / f a/b/c records     utils/mesh.py:28-79
      assets/pretrains/front_facial.json, front_face_1.json, head.json    {"face": [...]}   utils/mesh.py:214-245, 327-365
      assets/pretrains/smpl_part_info.json  {part: {"face": [...]}} x 10                utils/mesh.py:247-268
      assets/pretrains/smpl_model.pkl       protocol-2 pickle (keys of batch_smpl.py:236-283)
      assets/pretrains/hmr_tf2pt.pth        HumanModelRecovery.state_dict()             models/imitator.py:69-74
      outputs/checkpoints/G.pth             ImpersonatorGenerator.state_dict()          models/imitator.py:58-59
      src.png, targets/000.png ...          source / driving frames

    -> dict of paths.  Deterministic in ``seed``."""
    import json
    import os
    import pickle
    import cv2
    from .generator import ImpersonatorGenerator
    from .hmr import HumanModelRecovery
    pre = os.path.join(root, "assets", "pretrains")
    os.makedirs(pre, exist_ok=True)
    os.makedirs(os.path.join(root, "outputs", "checkpoints"), exist_ok=True)
    os.makedirs(os.path.join(root, "targets"), exist_ok=True)
    v, f = uv_sphere()
    np.save(os.path.join(pre, "smpl_faces.npy"), f.numpy())
    rs = np.random.RandomState(seed)
    nvt = 7576                                                     # SMPL's uv vertex count
    vts = rs.rand(nvt, 2)
    fvt = rs.randint(1, nvt + 1, size=(SMPL_F, 3))
    with open(os.path.join(pre, "mapper.txt"), "w") as fp:
        for p in v.numpy():
            fp.write("v %.6f %.6f %.6f\n" % tuple(p))
        fp.write("vn 0.0 0.0 1.0\n")
        for p in vts:
            fp.write("vt %.6f %.6f\n" % tuple(p))
        for tri, uv in zip(f.numpy() + 1, fvt):
            fp.write("f %d/%d/1 %d/%d/1 %d/%d/1\n" % (tri[0], uv[0], tri[1], uv[1], tri[2], uv[2]))
    head = sorted(rs.choice(SMPL_F, size=1200, replace=False).tolist())
    front = sorted(rs.choice(head, size=500, replace=False).tolist())
    json.dump({"face": front}, open(os.path.join(pre, "front_facial.json"), "w"))
    json.dump({"face": head}, open(os.path.join(pre, "head.json"), "w"))
    json.dump({"face": front}, open(os.path.join(pre, "front_face_1.json"), "w"))
    json.dump(synthetic_part_info(), open(os.path.join(pre, "smpl_part_info.json"), "w"))
    smpl = synthetic_smpl_model(seed=3)
    with open(os.path.join(pre, "smpl_model.pkl"), "wb") as fp:
        pickle.dump(smpl, fp, protocol=2)
    hmr = HumanModelRecovery(smpl_model=smpl)
    full = dict(hmr.state_dict())
    full.update(synthetic_hmr_state(hmr.state_dict()))
    torch.save(full, os.path.join(pre, "hmr_tf2pt.pth"))
    gen = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    gsd = fill_state_dict(gen.state_dict(), seed=0)
    torch.save({"module." + k if i % 2 else k: t for i, (k, t) in enumerate(gsd.items())},           # BaseModel._load_params strips it
               os.path.join(root, "outputs", "checkpoints", "G.pth"))

    def to_u8(img):                                               # [3,H,W] in [-1,1] -> BGR uint8 HWC
        a = ((img.permute(1, 2, 0).numpy() + 1) * 127.5).round().clip(0, 255).astype(np.uint8)
        return a[..., ::-1].copy()
    cv2.imwrite(os.path.join(root, "src.png"), to_u8(synthetic_source(image_size, seed=99)[0]))
    tgt = []
    for i in range(n_targets):
        pth = os.path.join(root, "targets", "%03d.png" % i)
        cv2.imwrite(pth, to_u8(synthetic_source(320, seed=200 + i)[0]))       # another size: the loaders resize
        tgt.append(pth)
    return dict(root=root, src=os.path.join(root, "src.png"), targets=os.path.join(root, "targets"), target_files=tgt,
                smpl_model=os.path.join(pre, "smpl_model.pkl"), hmr_model=os.path.join(pre, "hmr_tf2pt.pth"),
                load_path=os.path.join(root, "outputs", "checkpoints", "G.pth"), generator_state=gsd, hmr_state=full)
