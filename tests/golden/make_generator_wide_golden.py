"""Generates tests/golden/generator_wide.npz -- run ONLY where the reference checkout exists (/root/reference).

The generator conditioned on the wide maps of ``--map_name``: ImpersonatorGenerator(bg_dim=4, src_dim=tsf_dim=14) ('par',
11 conditioning channels) and 18 ('binary', 15), models/models.py:84-93.  Imports the reference's own
networks/generator.py (pure torch.nn; ipdb/h5py stubbed, as make_generator_golden.py does), loads the deterministic weights
of impersonator_b200.synthetic.fill_state_dict(seed=0) and, on synthetic_generator_inputs(..., cin=14 / 18), stores strided
slices of
  the src net's 7x7 stem before its InstanceNorm (networks/generator.py:80-84)      "<w>_stem_raw"
  encode_src                               (:213-214)    B=1                         "<w>_enc<i>", "<w>_res5"
  infer_front                              (:216-243)    B=1                         "<w>_front_*"
  encode_src + inference                   (:277-301)    B=2                         "<w>_inf_*"
  swap                                     (:245-275)    B=1, two sources            "<w>_swap_*"
at 256 x 256 for w = 14 and 18, and encode_src + inference for w = 18, B=1 at 512 x 512 ("w18_512_inf_*").

The LWB's grid_sample runs under make_generator_golden.torch12_grid_sample (the reference's pinned torch 1.2: the
flag-less call means align_corners=True).  oracle/generator_ref.py is checked against the reference modules on the full
tensors here (1e-5), so the slices pin both.

Byte-reproducible: one CPU thread (the fp32 convolutions then sum in a fixed order) and a zip archive written with fixed
entry times; run it twice and the files are identical.
"""
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_generator_golden import ImpersonatorGenerator, G, synthetic, torch12_grid_sample   # noqa: E402
from generator_wide_cases import WIDTHS, cases, feat, sl, stem_slice                        # noqa: E402


def check(name, a, b):
    d = (a - b).abs().max().item()
    print("%-22s restatement-vs-reference max-abs %.3g" % (name, d))
    assert d < 1e-5, name


def width(cin, out):
    net = ImpersonatorGenerator(bg_dim=4, src_dim=cin, tsf_dim=cin, repeat_num=6).eval()
    sd = synthetic.fill_state_dict(net.state_dict(), seed=0)
    net.load_state_dict(sd, strict=True)
    c = cases(cin)
    p = "w%d_" % cin

    src = c["front"]["src"]
    stem = torch.nn.functional.conv2d(src, sd["src_model.encoders.0.0.weight"], padding=3)
    check(p + "stem_raw", net.src_model.encoders[0][0](src), stem)
    out[p + "stem_raw"] = stem_slice(stem)
    enc, res = net.encode_src(src)
    e_m, r_m = G.encode_src(src, sd)
    for i in range(4):
        check(p + "enc%d" % i, enc[i], e_m[i])
        out[p + "enc%d" % i] = feat(enc[i])
    check(p + "res5", res[5], r_m[5])
    out[p + "res5"] = feat(res[5])

    f = c["front"]
    ref = net.infer_front(f["src"], f["tsf"], f["T"])
    mine = G.infer_front(f["src"], f["tsf"], f["T"], sd)
    for name, a, b in zip(("src_img", "src_mask", "tsf_img", "tsf_mask"), ref, mine):
        check(p + "front_" + name, a, b)
        out[p + "front_" + name] = sl(a)

    i2 = c["inf"]
    enc, res = net.encode_src(i2["src"])
    img, mask = net.inference([e.expand(2, -1, -1, -1) for e in enc], [e.expand(2, -1, -1, -1) for e in res],
                              i2["tsf"], i2["T"])
    e_m, r_m = G.encode_src(i2["src"], sd)
    img_m, mask_m = G.inference(e_m, r_m, i2["tsf"], i2["T"], sd)
    for name, a, b in (("inf_img", img, img_m), ("inf_mask", mask, mask_m)):
        check(p + name, a, b)
        out[p + name] = sl(a)

    a, b = c["swap_a"], c["swap_b"]
    e12, r12 = net.encode_src(a["src"])
    e21, r21 = net.encode_src(b["src"])
    s_img, s_mask = net.swap(a["tsf"], e12, e21, r12, r21, a["T"], b["T"])
    o12, q12 = G.encode_src(a["src"], sd)
    o21, q21 = G.encode_src(b["src"], sd)
    m_img, m_mask = G.swap(a["tsf"], o12, o21, q12, q21, a["T"], b["T"], sd)
    for name, x, y in (("swap_img", s_img, m_img), ("swap_mask", s_mask, m_mask)):
        check(p + name, x, y)
        out[p + name] = sl(x)

    if cin == 18:
        i5 = c["inf512"]
        enc, res = net.encode_src(i5["src"])
        img, mask = net.inference(enc, res, i5["tsf"], i5["T"])
        e_m, r_m = G.encode_src(i5["src"], sd)
        img_m, mask_m = G.inference(e_m, r_m, i5["tsf"], i5["T"], sd)
        for name, x, y in (("512_inf_img", img, img_m), ("512_inf_mask", mask, mask_m)):
            check(p + name, x, y)
            out[p + name] = sl(x, 16)


def save_npz(path, arrays):
    """np.savez_compressed with fixed entry times and order, so equal arrays give equal bytes."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    torch.set_grad_enabled(False)
    torch.set_num_threads(1)
    out = {}
    with torch12_grid_sample():
        for cin in WIDTHS:
            width(cin, out)
    path = os.path.join(HERE, "generator_wide.npz")
    save_npz(path, out)
    print("wrote", path, {k: v.shape for k, v in sorted(out.items())})


if __name__ == "__main__":
    main()
