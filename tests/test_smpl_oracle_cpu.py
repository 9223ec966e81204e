"""The SMPL oracle (oracle/smpl_ref.py) against outputs of the reference class networks.batch_smpl.SMPL
(tests/golden/smpl.npz, made by tests/golden/make_smpl_golden.py).  CPU only."""
import os

import numpy as np
import torch

from impersonator_b200 import synthetic as S
from oracle import smpl_ref

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "smpl.npz")


def golden_theta():
    theta = S.synthetic_smpl_params(5, seed=17)
    theta[1, 3:75] = 0
    return theta


def test_oracle_matches_reference_class():
    torch.set_grad_enabled(False)
    g = np.load(GOLD)
    m = smpl_ref.model_tensors(S.synthetic_smpl_model(seed=3))
    theta = golden_theta()
    for tag, rot in (("std", False), ("rot", True)):
        verts, joints, Rs, _ = smpl_ref.forward(m, theta[:, 75:].contiguous(), theta[:, 3:75].contiguous(), rotate_base=rot)
        assert np.abs(verts[:, ::13].numpy() - g["verts_" + tag]).max() < 2e-6
        assert np.abs(joints.numpy() - g["joints_" + tag]).max() < 2e-6
        assert np.abs(Rs.numpy() - g["Rs_" + tag]).max() < 1e-6
        j2d = smpl_ref.orth_proj_idrot(joints, theta[:, :3])
        assert np.abs(j2d.numpy() - g["j2d_" + tag]).max() < 2e-6


def test_float64_oracle_matches_reference_class():
    """The oracle run in float64 (the reference of the smpl_forward glue cases) meets the float32 golden of the reference
    class at the golden's own precision."""
    torch.set_grad_enabled(False)
    g = np.load(GOLD)
    m = smpl_ref.model_tensors(S.synthetic_smpl_model(seed=3))
    theta = golden_theta().double()
    for tag, rot in (("std", False), ("rot", True)):
        verts, joints, Rs, _ = smpl_ref.forward(m, theta[:, 75:].contiguous(), theta[:, 3:75].contiguous(), rotate_base=rot)
        assert verts.dtype == torch.float64
        assert np.abs(verts[:, ::13].numpy() - g["verts_" + tag]).max() < 2e-6
        assert np.abs(joints.numpy() - g["joints_" + tag]).max() < 2e-6
        assert np.abs(Rs.numpy() - g["Rs_" + tag]).max() < 1e-6
        j2d = smpl_ref.orth_proj_idrot(joints, theta[:, :3])
        assert np.abs(j2d.numpy() - g["j2d_" + tag]).max() < 2e-6


def test_rest_pose_is_shaped_template():
    """theta = 0: every rotation is the identity, so verts = v_template + shape blend (batch_smpl.py:312)."""
    torch.set_grad_enabled(False)
    m = smpl_ref.model_tensors(S.synthetic_smpl_model(seed=3))
    beta = torch.randn(2, 10, generator=torch.Generator().manual_seed(1))
    verts, _, Rs, _ = smpl_ref.forward(m, beta, torch.zeros(2, 72))
    v_shaped = (beta @ m["shapedirs"]).view(2, -1, 3) + m["v_template"]
    assert (Rs - torch.eye(3)).abs().max() < 1e-6
    assert (verts - v_shaped).abs().max() < 1e-5
