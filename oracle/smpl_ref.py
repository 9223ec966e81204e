"""ORACLE (test infrastructure only; never on the product path): CPU restatement in torch of the reference's
SMPL body model, ``networks/batch_smpl.py`` -- batch_rodrigues (:64-101), batch_global_rigid_transformation
(:129-218), batch_orth_proj_idrot (:221-233), SMPL.forward (:285-375) -- written functionally over a model
dict with the pickle's keys.  Pinned against the reference class itself by tests/golden/smpl.npz
(tests/golden/make_smpl_golden.py imports networks.batch_smpl from /root/reference)."""
import numpy as np
import torch


def model_tensors(dd):                                   # batch_smpl.py:236-283
    nb = dd['shapedirs'].shape[-1]
    return dict(
        v_template=torch.FloatTensor(np.asarray(dd['v_template'])),
        shapedirs=torch.FloatTensor(np.reshape(dd['shapedirs'], [-1, nb]).T.copy()),
        J_regressor=torch.FloatTensor(np.asarray(dd['J_regressor'].T.todense())),
        posedirs=torch.FloatTensor(np.reshape(dd['posedirs'], [-1, dd['posedirs'].shape[-1]]).T.copy()),
        parents=np.array(dd['kintree_table'][0].astype(np.int32)),
        weights=torch.FloatTensor(np.asarray(dd['weights'])),
        joint_regressor=torch.FloatTensor(np.asarray(dd['cocoplus_regressor'].T.todense())))


def rodrigues(theta):                                    # :64-101
    angle = torch.norm(theta + 1e-8, p=2, dim=1, keepdim=True)
    r = theta / angle
    c, s = torch.cos(angle)[..., None], torch.sin(angle)[..., None]
    outer = r[:, :, None] * r[:, None, :]
    z = torch.zeros_like(r[:, 0])
    skew = torch.stack([z, -r[:, 2], r[:, 1], r[:, 2], z, -r[:, 0], -r[:, 1], r[:, 0], z], dim=1).view(-1, 3, 3)
    return c * torch.eye(3, dtype=theta.dtype)[None] + (1 - c) * outer + s * skew


def rigid_chain(Rs, Js, parents, rotate_base=False):    # :129-218
    N = Rs.shape[0]
    root = Rs[:, 0]
    if rotate_base:
        root = root @ torch.diag(torch.tensor([1., -1., -1.], dtype=Rs.dtype))

    def make_A(R, t):
        top = torch.cat([R, t[:, :, None]], dim=2)
        return torch.cat([top, torch.tensor([0., 0., 0., 1.], dtype=R.dtype).expand(N, 1, 4)], dim=1)

    res = [make_A(root, Js[:, 0])]
    for i in range(1, parents.shape[0]):
        res.append(res[parents[i]] @ make_A(Rs[:, i], Js[:, i] - Js[:, parents[i]]))
    res = torch.stack(res, dim=1)
    new_J = res[:, :, :3, 3]
    init_bone = res @ torch.cat([Js, Js.new_zeros(N, 24, 1)], dim=2)[..., None]
    A = res - torch.nn.functional.pad(init_bone, (3, 0))
    return new_J, A


def forward(m, beta, theta, rotate_base=False):          # :285-375 -> verts, joints, Rs, J_transformed
    """In the dtype of beta / theta: model tensors of another float dtype are cast (float64 runs the oracle as a
    float64 reference of the kernel)."""
    m = {k: (v.to(beta.dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in m.items()}
    N = beta.shape[0]
    V = m['v_template'].shape[0]
    v_shaped = (beta @ m['shapedirs']).view(N, V, 3) + m['v_template']
    J = torch.stack([v_shaped[:, :, d] @ m['J_regressor'] for d in range(3)], dim=2)
    Rs = rodrigues(theta.reshape(-1, 3)).view(N, 24, 3, 3)
    pose_feature = (Rs[:, 1:] - torch.eye(3, dtype=Rs.dtype)).reshape(N, 207)
    v_posed = (pose_feature @ m['posedirs']).view(N, V, 3) + v_shaped
    J_transformed, A = rigid_chain(Rs, J, m['parents'], rotate_base)
    T = (m['weights'][None].expand(N, -1, -1) @ A.view(N, 24, 16)).view(N, V, 4, 4)
    v_h = torch.cat([v_posed, v_posed.new_ones(N, V, 1)], dim=2)[..., None]
    verts = (T @ v_h)[:, :, :3, 0]
    joints = torch.stack([verts[:, :, d] @ m['joint_regressor'] for d in range(3)], dim=2)
    return verts, joints, Rs, J_transformed


def orth_proj_idrot(X, camera):                          # :221-233
    return camera[:, None, 0:1] * (X[:, :, :2] + camera[:, None, 1:])


def get_details(m, theta):                               # networks/hmr.py:302-330
    cam, pose, shape = theta[:, 0:3].contiguous(), theta[:, 3:75].contiguous(), theta[:, 75:].contiguous()
    verts, j3d, Rs, _ = forward(m, shape, pose)
    return dict(theta=theta, cam=cam, pose=pose, shape=shape, verts=verts, j2d=orth_proj_idrot(j3d, cam), j3d=j3d)
