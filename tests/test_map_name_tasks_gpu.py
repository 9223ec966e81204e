"""``Imitator(opt)``, ``Viewer(opt)`` and ``Swapper(opt)`` with ``opt.map_name`` other than the default 'uv_seg': the
generator is built for 3 + get_map_fn_dim(map_name) input channels and its checkpoint loaded from a file, the renderer's
conditioning table comes from mesh.create_mapping(map_name) on synthetic asset files in the real formats
(synthetic.write_synthetic_assets).  'par' (14 generator input channels) and 'binary' (18) run the wide row-K stem;
'seg', 'uv' (4, 5) and 'ids' (4) the 8-channel one.  Checked against the CPU oracle (oracle/tasks_ref.py): the
conditioning maps bit for bit, the frames at the 1e-3 max-abs bar."""
import os

import numpy as np
import pytest
import torch

import tasks_common as C
from impersonator_b200 import mesh
from impersonator_b200 import synthetic as S
from impersonator_b200.generator import ImpersonatorGenerator
from oracle import tasks_ref as T

pytestmark = pytest.mark.gpu
TOL = 1e-3


@pytest.fixture(scope="module")
def assets(cuda, tmp_path_factory):
    torch.set_grad_enabled(False)
    root = str(tmp_path_factory.mktemp("map_name_assets"))
    A = S.write_synthetic_assets(root)
    a_png, b_png = C.write_inputs(root)
    v, f = S.uv_sphere()
    return dict(root=root, A=A, a=a_png, b=b_png, v=v, f=f, g=np.load(C.GOLD), nets={})


def checkpoint(assets, map_name):
    """-> (load_path, state_dict) of a seeded generator for map_name's input width, saved like a trained checkpoint."""
    if map_name not in assets["nets"]:
        cin = 3 + mesh.get_map_fn_dim(map_name)
        net = ImpersonatorGenerator(bg_dim=4, src_dim=cin, tsf_dim=cin, repeat_num=6)
        sd = S.fill_state_dict(net.state_dict(), seed=0)
        path = os.path.join(assets["root"], "outputs", "checkpoints", "G_%s.pth" % map_name)
        torch.save(sd, path)
        assets["nets"][map_name] = (path, sd)
    return assets["nets"][map_name]


def make_opt(assets, map_name, front=False):
    opt = C.Opt()
    opt.map_name, opt.front_warp = map_name, front
    opt.load_path = checkpoint(assets, map_name)[0]
    return opt


def tables(map_name):
    """The oracle's tables, from the same asset files (cwd = the asset root)."""
    mp = "assets/pretrains/mapper.txt"
    t = lambda a: torch.as_tensor(np.asarray(a)).float()          # noqa: E731
    return dict(map_fn=t(mesh.create_mapping(map_name, mp, contain_bg=True, fill_back=False)),
                front_map_fn=t(mesh.create_mapping('front', mp, contain_bg=True, fill_back=False)),
                back_map_fn=t(mesh.create_mapping('back', mp, contain_bg=True, fill_back=False)))


def oracle_info(assets, png, theta, tabs, sd, task, part_fn=None):
    d = S.QuarterTurnBodyModel(assets["v"]).get_details(torch.from_numpy(theta)[None])
    return T.personalize(C.read_like_reference(png), d["cam"], d["verts"], assets["f"], tabs, sd, C.SIZE, task, part_fn)


@pytest.mark.parametrize("map_name", ["par", "binary", "seg", "uv", "ids"])
def test_imitator_personalize_and_inference(cuda, assets, monkeypatch, map_name):
    from impersonator_b200.imitator import Imitator
    monkeypatch.chdir(assets["root"])
    g = assets["g"]
    im = Imitator(make_opt(assets, map_name), hmr=S.QuarterTurnBodyModel(assets["v"]), device=cuda)
    width = mesh.get_map_fn_dim(map_name)
    assert im.render.map_fn.shape == (S.SMPL_F + 1, width)
    assert im.generator.tsf_model.encoders[0][0].weight.shape[1] == 3 + width
    im.personalize(assets["a"], src_smpl=g["src_theta"].copy())
    _, sd = checkpoint(assets, map_name)
    tabs = tables(map_name)
    info = oracle_info(assets, assets["a"], g["src_theta"], tabs, sd, "imitator")
    assert torch.equal(im.src_info["cond"].cpu(), info["cond"]), "conditioning map differs from the oracle"
    thetas = [th.copy() for th in g["imit_thetas"]]
    frames = im.inference_by_smpls(thetas, cam_strategy="smooth")
    shape = torch.from_numpy(g["src_theta"][None, -10:]).float()
    ref, _ = T.imitate(info, shape, torch.from_numpy(np.stack(thetas)).float(), S.QuarterTurnBodyModel(assets["v"]),
                       assets["f"], tabs, sd, C.SIZE, cam_strategy="smooth")
    errs = [float(np.abs(a - b).max()) for a, b in zip(frames, ref)]
    print("Imitator map_name=%s vs oracle: %s" % (map_name, ["%.2e" % e for e in errs]))
    assert len(frames) == len(ref) == len(thetas) and max(errs) < TOL


@pytest.mark.parametrize("map_name", ["par", "binary"])
def test_viewer_view(cuda, assets, monkeypatch, map_name):
    from impersonator_b200.viewer import Viewer
    monkeypatch.chdir(assets["root"])
    g = assets["g"]
    vw = Viewer(make_opt(assets, map_name, front=True), hmr=S.QuarterTurnBodyModel(assets["v"]), device=cuda)
    vw.personalize(assets["a"], src_smpl=g["src_theta"].copy())
    _, sd = checkpoint(assets, map_name)
    tabs = tables(map_name)
    info = oracle_info(assets, assets["a"], g["src_theta"], tabs, sd, "viewer")
    assert torch.equal(vw.src_info["cond"].cpu(), info["cond"])
    rt, t = g["views"][0]
    preds = vw.view(rt / 180 * np.pi, t)
    c = T.nmr_ref.correspond(info["cam"], vw.tsf_info["verts"].cpu(), assets["f"], tabs["map_fn"], info["p2verts"],
                             info["img"], C.SIZE)
    ref, _, mask = T.G.imitator_forward(torch.zeros_like(info["bg"]), info["feats"], c["tsf_inputs"], c["T"], sd)
    fm = T.nmr_ref.encode_fim(c["fim"], tabs["front_map_fn"])
    ref = (1 - fm) * ref + c["tsf_img"] * fm * (1 - mask)
    e = (preds.cpu() - ref).abs().max().item()
    print("Viewer map_name=%s (front_warp) vs oracle: %.2e" % (map_name, e))
    assert e < TOL


@pytest.mark.parametrize("map_name", ["par", "binary"])
def test_swapper_swap(cuda, assets, monkeypatch, map_name):
    from impersonator_b200.swapper import Swapper
    monkeypatch.chdir(assets["root"])
    g = assets["g"]
    sw = Swapper(make_opt(assets, map_name), hmr=S.QuarterTurnBodyModel(assets["v"]), device=cuda)
    assert sw.part_fn.shape == (S.SMPL_F + 1, 11)                     # the part table stays 'par' whatever the map
    sw.swap_setup(assets["a"], assets["b"], src_smpl=g["src_theta"].copy(), tgt_smpl=g["tgt_theta"].copy())
    _, sd = checkpoint(assets, map_name)
    tabs = tables(map_name)
    part_fn = sw.part_fn.cpu()
    part_faces = list(mesh.get_part_face_ids('par', "assets/pretrains/mapper.txt", fill_back=False).values())
    infos = [oracle_info(assets, png, g[key], tabs, sd, "swapper", part_fn)
             for png, key in ((assets["a"], "src_theta"), (assets["b"], "tgt_theta"))]
    assert torch.equal(sw.src_info["cond"].cpu(), infos[0]["cond"])
    preds = sw.swap(sw.src_info, sw.tsf_info, target_part="body")
    ref, _, _ = T.swap(infos[0], infos[1], part_faces, tabs, sd, C.SIZE, "body")
    e = (preds.cpu() - ref).abs().max().item()
    print("Swapper map_name=%s vs oracle: %.2e" % (map_name, e))
    assert e < TOL
