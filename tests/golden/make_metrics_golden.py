"""Generates tests/golden/metrics.npz on a CPU host with the reference checkout:

    python tests/golden/make_metrics_golden.py <reference checkout>

LPIPS: builds the reference's own PNetLin(pnet_type='alex', version='0.1') from his_evaluators/metrics/lpips/models/
(networks_basic.py, pretrained_networks.py) with pretrained=False, loads the seeded synthetic AlexNet and `lin` weights
of tests/metrics_cases.py into it, and stores its scores and per-layer values in float64 for every case.  Only
networks_basic's module-level imports need stand-ins here: skimage (not installed; util.py imports compare_ssim, which
PNetLin never calls) and torchvision's alexnet(pretrained=...) keyword, which torchvision 0.26 spells weights=None.

SSIM / PSNR: skimage is not installed, so the stored values are those of oracle/metrics_ref.py; tests/test_metrics_cpu.py
pins that restatement to hand-worked cases.

Inputs are regenerated from their seeds; the golden stores their SHA-256.  The archive is written with fixed zip
timestamps, so rerunning the script reproduces it byte for byte."""
import io
import os
import sys
import types
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import metrics_cases as MC                                              # noqa: E402
from oracle import metrics_ref as R                                     # noqa: E402

LPIPS_DIR = os.path.join("thirdparty", "his_evaluators", "his_evaluators", "metrics", "lpips")
OUT = os.path.join(HERE, "metrics.npz")


def save_npz(path, arrays):
    """np.savez_compressed with a fixed member timestamp and order."""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            b = io.BytesIO()
            np.lib.format.write_array(b, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            z.writestr(info, b.getvalue())
    with open(path, "wb") as f:
        f.write(buf.getvalue())


def reference_pnetlin(ref_root, convs, lins):
    sk = types.ModuleType("skimage")
    sk.measure = types.ModuleType("skimage.measure")
    sk.measure.compare_ssim = None
    sys.modules.setdefault("skimage", sk)
    sys.modules.setdefault("skimage.measure", sk.measure)
    import torchvision.models as tvm
    alexnet = tvm.alexnet
    tvm.alexnet = lambda pretrained=False, **kw: alexnet(weights=None, **kw)
    pkg = types.ModuleType("lpips")                                     # the package without its __init__ (dist_model)
    pkg.__path__ = [os.path.join(ref_root, LPIPS_DIR)]
    sys.modules["lpips"] = pkg
    from lpips.models import networks_basic as nb
    net = nb.PNetLin(pnet_type='alex', pnet_rand=True, use_gpu=False, version='0.1')
    tvm.alexnet = alexnet
    feats = net.net[0]
    mods = [feats.slice1[0], feats.slice2[1], feats.slice3[1], feats.slice4[0], feats.slice5[0]]
    with torch.no_grad():
        for m, (w, b) in zip(mods, convs):
            m.weight.copy_(w)
            m.bias.copy_(b)
    net.load_state_dict(MC.lin_state_dict(lins))
    net.eval()
    net.net[0].double()
    net.double()
    return net


def main():
    torch.set_grad_enabled(False)
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    net = reference_pnetlin(sys.argv[1], convs, lins)
    g = dict(weights_sha=np.array(MC.sha256(*[t for wb in convs for t in wb], *lins)))
    for name in MC.CASES:
        preds, gts = MC.make_case(name)
        g[name + "/sha"] = np.array(MC.sha256(preds, gts))
        g[name + "/ssim"] = R.ssim_scores(preds, gts)
        g[name + "/psnr"] = R.psnr_scores(preds, gts)
        p = torch.from_numpy(preds) * 2 - 1                             # PerceptualMetric.preprocess, float32
        t = torch.from_numpy(gts) * 2 - 1
        val = net.forward(t.double(), p.double())                       # forward_pair(target, pred)
        net.spatial = True
        maps = net.forward(t.double(), p.double())
        net.spatial = False
        g[name + "/lpips"] = val.view(-1).numpy()
        g[name + "/lpips_layers"] = torch.stack([m.mean(dim=(2, 3))[:, 0] for m in maps], dim=1).numpy()
        print(name, g[name + "/ssim"][:2], g[name + "/psnr"][:2], g[name + "/lpips"][:2])
    scores = [net.forward((torch.from_numpy(gt) * 2 - 1).double(), (torch.from_numpy(pr) * 2 - 1).double())
              for pr, gt in [(a[i:i + 32], b[i:i + 32]) for a, b in [MC.make_case("batch33")] for i in (0, 32)]]
    g["batch33/calculate_score"] = np.array(torch.stack([s.double().mean() for s in scores]).mean().item())
    save_npz(OUT, g)


if __name__ == "__main__":
    main()
