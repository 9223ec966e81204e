"""TEST INFRASTRUCTURE ONLY -- torch-CPU restatement of the geometry glue around the rasterizer.

Follows, line by line (device-agnostic torch code of the reference with ``.cuda()`` removed):
  utils/nmr.py:10-28      orthographic_proj_withz_idrot
  utils/nmr.py:263-278    SMPLRenderer.render_fim_wim   (y flip :271, look_at :273, gather :276)
  thirdparty/neural_renderer/neural_renderer/look_at.py:48-60    (R == I for eye = [0,0,-(1/tan30+1)])
  thirdparty/neural_renderer/neural_renderer/vertices_to_faces.py:17-21
  utils/nmr.py:328-341    encode_fim  (map_fn[fim.long()], fim == -1 -> last row)
  utils/nmr.py:617-659    cal_bc_transform
  models/imitator.py:105-107  src p2verts = f2verts[..., :2] with y negated
  utils/nmr.py:343-352    encode_front_fim;  utils/nmr.py:506-546  get_vis_f2pts
The rasterizer itself is oracle/raster.py (C restatement / reference CUDA).
No reference TEST pins these (SURVEY 8c), so the restatement is pinned to the reference's CODE:
tests/golden/make_nmr_golden.py imports /root/reference/utils/nmr.py unmodified, calls the
``SMPLRenderer`` methods above as unbound functions and asserts torch.equal against every function
here; the committed tests/golden/nmr.npz carries those outputs to the CPU suite and the GPU box.
Tolerance of the CUDA path vs this file: fim exact, wim/cond/T 1e-5.

``align_corners``: the reference calls F.grid_sample without the flag (networks/generator.py:313,
models/imitator.py:259) under its pinned torch==1.2.0 (requirements.txt:6), where that means
align_corners=True -- the default here; False (= what the installed torch 2.11 does for the same
call) is the opt-in.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from . import raster

EYE_Z = -(1. / np.tan(np.radians(30)) + 1)     # utils/nmr.py:177


def orthographic_proj_withz_idrot(X, cam, offset_z=0.):       # utils/nmr.py:10-28
    scale = cam[:, 0].contiguous().view(-1, 1, 1)
    trans = cam[:, 1:3].contiguous().view(cam.size(0), 1, -1)
    proj_xy = scale * (X[:, :, :2] + trans)
    proj_z = X[:, :, 2, None] + offset_z
    return torch.cat((proj_xy, proj_z), 2)


def look_at(vertices, eye):                                    # look_at.py:6-62 (batched cross with dim=-1)
    eye = torch.tensor(eye, dtype=torch.float32)
    at = torch.tensor([0, 0, 0], dtype=torch.float32)
    up = torch.tensor([0, 1, 0], dtype=torch.float32)
    bs = vertices.shape[0]
    eye = eye[None, :].repeat(bs, 1)
    at = at[None, :].repeat(bs, 1)
    up = up[None, :].repeat(bs, 1)
    z_axis = F.normalize(at - eye, eps=1e-5)
    x_axis = F.normalize(torch.linalg.cross(up, z_axis, dim=-1), eps=1e-5)
    y_axis = F.normalize(torch.linalg.cross(z_axis, x_axis, dim=-1), eps=1e-5)
    r = torch.cat((x_axis[:, None, :], y_axis[:, None, :], z_axis[:, None, :]), dim=1)
    vertices = vertices - eye[:, None, :]
    return torch.matmul(vertices, r.transpose(1, 2))


def vertices_to_faces(vertices, faces):                        # vertices_to_faces.py:4-22
    bs, nv = vertices.shape[:2]
    faces = faces + (torch.arange(bs, dtype=torch.int32) * nv)[:, None, None]
    vertices = vertices.reshape((bs * nv, 3))
    return vertices[faces.long()]


def project_to_faces(cam, vertices, faces_idx):
    """utils/nmr.py:263-276 up to (not including) the rasterizer: f32 [B,F,3,3]."""
    bs = cam.shape[0]
    faces = faces_idx.int()[None].repeat(bs, 1, 1)
    proj_verts = orthographic_proj_withz_idrot(vertices, cam)
    proj_verts[:, :, 1] *= -1
    verts = look_at(proj_verts, [0, 0, EYE_Z])
    return vertices_to_faces(verts, faces)


def render_fim_wim(cam, vertices, faces_idx, image_size, near=0.1, far=100.0):
    """SMPLRenderer.render_fim_wim (utils/nmr.py:263-278) -> f2verts, fim, wim (torch CPU).  near / far: the nr
    defaults, which the reference's renderer passes."""
    f2verts = project_to_faces(cam, vertices, faces_idx)
    fim, wim, _ = raster.rasterize_fim_wim(f2verts.numpy(), image_size, near, far)
    return f2verts, torch.from_numpy(fim), torch.from_numpy(wim)


def encode_fim(fim, map_fn, transpose=True):                  # utils/nmr.py:328-341
    fim_enc = map_fn[fim.long()]
    if transpose:
        fim_enc = fim_enc.permute(0, 3, 1, 2)
    return fim_enc


def src_p2verts(f2verts):                                      # models/imitator.py:105-107
    p = f2verts[:, :, :, 0:2].clone()
    p[:, :, :, 1] *= -1
    return p


def cal_bc_transform(src_f2pts, dst_fims, dst_wims, image_size):   # utils/nmr.py:617-659
    bs = src_f2pts.shape[0]
    T = -2 * torch.ones((bs, image_size * image_size, 2), dtype=torch.float32)
    for i in range(bs):
        from_faces_verts_on_img = src_f2pts[i]
        to_face_index_map = dst_fims[i].long().reshape(-1)
        to_weight_map = dst_wims[i].reshape(-1, 3)
        to_exist_mask = (to_face_index_map != -1)
        to_exist_face_idx = to_face_index_map[to_exist_mask]
        to_exist_face_weights = to_weight_map[to_exist_mask]
        exist_smpl_T = (from_faces_verts_on_img[to_exist_face_idx] * to_exist_face_weights[:, :, None]).sum(dim=1)
        T[i, to_exist_mask] = exist_smpl_T
    return T.view(bs, image_size, image_size, 2)


def get_vis_f2pts(f2pts, fims):                                # utils/nmr.py:506-546
    def get_vis(orig_f2pts, fim):
        vis_f2pts = torch.zeros_like(orig_f2pts) - 2.0
        face_ids = fim.unique()[1:].long()                     # :528 drops the first unique value (assumed -1)
        vis_f2pts[face_ids] = orig_f2pts[face_ids]
        return vis_f2pts
    if f2pts.dim() == 4:
        return torch.stack([get_vis(f2pts[i], fims[i]) for i in range(f2pts.shape[0])], dim=0)
    return get_vis(f2pts, fims)


def grid_sample(x, T, align_corners=True):
    """F.grid_sample(x, T) as the reference calls it (no flag: networks/generator.py:313,
    models/imitator.py:259): align_corners=True under the reference's torch 1.2."""
    return F.grid_sample(x, T, mode='bilinear', padding_mode='zeros', align_corners=align_corners)


def correspond(cam, vertices, faces_idx, map_fn, src_p2v, src_img, image_size, align_corners=True, near=0.1, far=100.0):
    """models/imitator.py:251-260 (transfer_params_by_smpl) for a batch of target frames whose
    source-side tables have batch 1 (or one per frame): returns dict(fim, wim, cond, T, tsf_img, tsf_inputs, f2verts)."""
    bs = cam.shape[0]
    f2verts, fim, wim = render_fim_wim(cam, vertices, faces_idx, image_size, near, far)
    cond = encode_fim(fim, map_fn)
    T = cal_bc_transform(src_p2v.expand(bs, -1, -1, -1), fim, wim, image_size)
    tsf_img = grid_sample(src_img.expand(bs, -1, -1, -1), T, align_corners)
    tsf_inputs = torch.cat([tsf_img, cond], dim=1)
    return dict(f2verts=f2verts, fim=fim, wim=wim, cond=cond, T=T, tsf_img=tsf_img, tsf_inputs=tsf_inputs)
