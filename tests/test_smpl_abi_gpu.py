"""lwb_smpl_forward through the raw C ABI: every output and the workspace are views inside sentinel bands that must
come back unchanged, and each nullable output (Rs, J_transformed, joints with j2d, j2d) passed as NULL in turn leaves
the other outputs byte-identical to the full call."""
import pytest
import torch

import glue_cases as G
from impersonator_b200._lib import check, lib, ptr, stream
from conv_emulation import assert_bands_intact, guarded

pytestmark = pytest.mark.gpu

B, V, NB = 9, 33, 10                     # frames 0..7 and a second FB = 8 pass of one; 32 vertices + a tail of one


def _call(cuda, model, beta, theta, cam, omit):
    nj = model["joint_regressor_t"].shape[0]
    shapes = dict(verts=(B, V, 3), joints=(B, nj, 3), Rs=(B, 24, 3, 3), Jt=(B, 24, 3), j2d=(B, nj, 2))
    bufs, outs = {}, {}
    for k, shape in shapes.items():
        if k in omit:
            continue
        bufs[k], outs[k] = guarded(cuda, shape, torch.float32, float("nan"))
    nws = lib().lwb_smpl_workspace_bytes(B)
    bufs["workspace"], ws = guarded(cuda, (nws,), torch.uint8, 0)
    check(lib().lwb_smpl_forward(
        ptr(beta), ptr(theta), B, NB, V, ptr(model["v_template"]), ptr(model["shapedirs"]), ptr(model["posedirs"]),
        ptr(model["j_template"]), ptr(model["j_shapedirs"]), ptr(model["parents"]), ptr(model["weights"]),
        ptr(model["joint_regressor_t"]), nj, 1, ptr(outs["verts"]), ptr(outs.get("joints")), ptr(outs.get("Rs")),
        ptr(outs.get("Jt")), ptr(cam if "j2d" in outs else None), ptr(outs.get("j2d")), ptr(ws), stream()),
        "lwb_smpl_forward")
    torch.cuda.synchronize()
    for k, buf in bufs.items():
        assert_bands_intact("%s (omitted %s)" % (k, ",".join(omit) or "none"), buf)
    return {k: v.cpu() for k, v in outs.items()}


@pytest.mark.parametrize("omit", [("Rs",), ("Jt",), ("j2d",), ("joints", "j2d")], ids=lambda o: "+".join(o))
def test_smpl_abi_null_outputs(cuda, omit):
    g = torch.Generator().manual_seed(2001)
    model = {k: t.to(cuda) for k, t in G.smpl_device_model(G.smpl_model(2001, V, NB)).items()}
    beta = (torch.randn(B, NB, generator=g)).to(cuda)
    theta = (torch.randn(B, 72, generator=g) * 0.4).to(cuda)
    cam = torch.cat([torch.rand(B, 1, generator=g) + 0.5, torch.randn(B, 2, generator=g) * 0.2], dim=1).to(cuda)
    full = _call(cuda, model, beta, theta, cam, ())
    for k, v in full.items():
        assert not torch.isnan(v).any(), "%s: the full call left sentinel NaNs" % k
    part = _call(cuda, model, beta, theta, cam, omit)
    assert set(part) == set(full) - set(omit)
    for k, v in part.items():
        assert torch.equal(v.view(torch.int32), full[k].view(torch.int32)), "%s differs when %s is NULL" % (k, omit)
