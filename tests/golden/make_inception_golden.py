"""Generates tests/golden/inception.npz on a CPU host with the reference checkout:

    python tests/golden/make_inception_golden.py <reference checkout>

Runs the reference's own his_evaluators/metrics/metrics.py in float64: its InceptionV3 wrapper (output_blocks=[3],
resize_input=False, normalize_input=False, as register_model builds it), FIDMetric / InceptionScoreMetric.preprocess,
forward and calculate_score, and BaseMetric.fid_score_func / is_score_func.  Stand-ins, each for something this host
cannot run as the reference wrote it:
  - skimage is not installed: an empty module (the IS / FID code never calls it);
  - inception_v3(pretrained=True) downloads ImageNet weights: torchvision's inception_v3(weights=None,
    init_weights=False), then the seeded synthetic weights of tests/inception_cases.py;
  - linalg.sqrtm(..., disp=False) raises TypeError on scipy >= 1.16: a shim that returns (sqrtm(A), None).

The BatchNorm running statistics are calibrated once: every BatchNorm is reset with momentum=None and the seeded
calibration batch runs through the wrapper in train mode, which leaves each layer's batch mean and unbiased variance as
its running statistics.  They are rounded to float32, stored (bn/<name>/mean|var) and used for every case.

Where the reference's FID raises (a rank-deficient product whose sqrtm has imaginary parts: 33 frames in
2048 dimensions), the golden stores NaN; every FID also has an `fid_eig` twin, oracle/inception_ref.py's eigenvalue
route on the same (reference) features.

Frames are passed as float64, so preprocess (x * 2 - 1, bilinear resize) runs in float64.  Inputs are regenerated from
their seeds; the golden stores their SHA-256.  The archive is written with fixed zip timestamps, so rerunning the script
reproduces it byte for byte."""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import inception_cases as IC                                            # noqa: E402
from oracle import inception_ref as R                                   # noqa: E402
from make_metrics_golden import save_npz                                # noqa: E402

METRICS_PY = os.path.join("thirdparty", "his_evaluators", "his_evaluators", "metrics", "metrics.py")
OUT = os.path.join(HERE, "inception.npz")


def reference_metrics(ref_root):
    """The reference's metrics.py as a module, with the stand-ins above."""
    sk = types.ModuleType("skimage")
    sk.metrics = types.ModuleType("skimage.metrics")
    sys.modules.setdefault("skimage", sk)
    sys.modules.setdefault("skimage.metrics", sk.metrics)
    import torchvision.models.inception as tvi
    made = []
    orig = tvi.inception_v3

    def inception_v3(pretrained=False, **kw):
        made.append(orig(weights=None, init_weights=False, **kw))
        return made[-1]

    tvi.inception_v3 = inception_v3
    spec = importlib.util.spec_from_file_location("his_metrics", os.path.join(ref_root, METRICS_PY))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    tvi.inception_v3 = orig
    from scipy import linalg

    def sqrtm(a, disp=True):
        return (linalg.sqrtm(a), None) if not disp else linalg.sqrtm(a)

    mod.linalg = types.SimpleNamespace(sqrtm=sqrtm)
    return mod, made


def reference_fid(fn):
    """The reference's FID, or NaN where its sqrtm of a rank-deficient product has imaginary parts beyond its 1e-3
    tolerance and calculate_frechet_distance raises ValueError ('Imaginary component ...')."""
    try:
        return np.array(float(fn()))
    except ValueError as e:
        print("reference raises:", e)
        return np.array(np.nan)


def main():
    torch.set_grad_enabled(False)
    mod, made = reference_metrics(sys.argv[1])
    net = mod.InceptionV3(output_blocks=[3], resize_input=False, normalize_input=False, requires_grad=False)
    inception = made[-1]
    params = IC.synthetic_inception()
    ones = {k + s: np.ones(v[0].shape[0], np.float32) for k, v in params.items() for s in ("/mean", "/var")}
    missing, unexpected = inception.load_state_dict(IC.state_dict(params, ones), strict=False)
    assert not unexpected and all(k.startswith(("AuxLogits.", "fc.")) or k.endswith("num_batches_tracked")
                                  for k in missing), missing
    net.double()
    bns = {name: inception.get_submodule(name + ".bn") for name in params}
    for bn in bns.values():
        bn.reset_running_stats()
        bn.momentum = None
    net.train()
    calib = IC.make_frames(*IC.CALIB)
    fid = mod.FIDMetric.__new__(mod.FIDMetric)
    mod.BaseMetric.__init__(fid, torch.device("cpu"))
    fid.height, fid.width = 299, 299
    net(fid.preprocess(torch.from_numpy(calib).double()))
    g = dict(calib_sha=np.array(IC.sha256(calib)),
             weights_sha=np.array(IC.sha256(*[t for p in params.values() for t in p])))
    for name, bn in bns.items():
        for k, buf in (("mean", bn.running_mean), ("var", bn.running_var)):
            g["bn/%s/%s" % (name, k)] = buf.float().numpy()
            buf.copy_(buf.float().double())
    net.eval()

    mod.MODEL_ZOOS[mod.BaseMetric.INCEPTION_V3] = net                   # register_model finds it: one shared model
    fid = mod.FIDMetric(torch.device("cpu"))
    ism = mod.InceptionScoreMetric(torch.device("cpu"))
    for name in IC.CASES:
        frames = IC.make_case(name)
        g[name + "/sha"] = np.array(IC.sha256(frames))
        g[name + "/feats"] = fid.forward(torch.from_numpy(frames).double())
        print(name, g[name + "/feats"].shape, np.abs(g[name + "/feats"]).max())
    preds, gts = IC.make_batch33()
    g["batch33/sha"] = np.array(IC.sha256(preds, gts))
    p64, t64 = torch.from_numpy(preds).double(), torch.from_numpy(gts).double()
    g["batch33/fid"] = reference_fid(lambda: fid.calculate_score(p64, t64))
    pf = np.concatenate([fid.forward(x[i:i + 32]) for x in (p64, t64) for i in (0, 32)])
    g["batch33/fid_eig"] = np.array(R.fid_eig(pf[:33], pf[33:]))
    g["batch33/is"] = np.array([float(v) for v in ism.calculate_score(p64)])
    print("batch33", g["batch33/fid"], g["batch33/fid_eig"], g["batch33/is"])
    for name in IC.FEATS:
        a, b = IC.make_feats(name)
        g["feats/%s/sha" % name] = np.array(IC.sha256(a, b))
        g["feats/%s/fid" % name] = reference_fid(lambda: mod.BaseMetric.fid_score_func(a, b))
        g["feats/%s/fid_eig" % name] = np.array(R.fid_eig(a, b))
        probs = torch.softmax(torch.from_numpy(a) * IC.IS_GAIN, dim=1).numpy()
        g["feats/%s/is" % name] = np.array(float(mod.BaseMetric.is_score_func(probs)))
        print(name, g["feats/%s/fid" % name], g["feats/%s/is" % name])
    save_npz(OUT, g)


if __name__ == "__main__":
    main()
