"""Image quality of the generator's operand modes against fp16x3, on the synthetic bench workload.

    python tools/precision_quality.py [--size 256] [--batch 16] [--sets 4] [--alexnet PATH] [--lin PATH]

Runs bench.py's imitation workload (synthetic generator weights, source and SMPL frames) with the generator pinned to
fp16x3, fp16f8 and fp16 and scores every frame of each mode against the fp16x3 frame of the same target on the device
(impersonator_b200.metrics: SSIM, PSNR, LPIPS).  LPIPS uses torchvision's AlexNet and his_evaluators' lin weights when
both paths are given; otherwise it runs on the seeded synthetic weights of the metric tests and is reported as
``lpips_synthetic``, which is a feature-space distance and not the perceptual metric.  Prints one JSON line with the
card name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--sets", type=int, default=4)
    ap.add_argument("--alexnet", default=None)
    ap.add_argument("--lin", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from detector_bench import card
    from impersonator_b200 import _lib, metrics as M, synthetic as S
    from impersonator_b200.generator import ImpersonatorGenerator
    from impersonator_b200.hmr import HumanModelRecovery
    from impersonator_b200.imitator import Imitator
    from impersonator_b200.nmr import SMPLRenderer

    _lib.require_gpu()
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    size, B = args.size, args.batch
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    net = net.to(dev).eval()
    render = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"], has_front=False).to(dev)

    class Opt(object):
        image_size, batch_size, bg_model, repeat_num, cond_nc = size, B, "ORIGINAL", 6, 3
        bg_ks, ft_ks, front_warp, only_vis = 13, 3, False, False
    body = HumanModelRecovery(smpl_model=S.synthetic_smpl_model(seed=3)).to(dev)
    imitator = Imitator(Opt(), generator=net, hmr=body, render=render, device=dev)
    src_img = S.synthetic_source(size)
    src_theta = S.synthetic_smpl_params(1, seed=5)[0]
    sets = [S.synthetic_smpl_params(B, seed=1000 + i) for i in range(args.sets)]

    if args.alexnet and args.lin:
        lp, lp_key = M.LPIPS(dev, weights=args.alexnet, lin_weights=args.lin), "lpips"
    else:
        import metrics_cases as MC
        lp = M.LPIPS(dev, weights=MC.alexnet_state_dict(MC.synthetic_alexnet()),
                     lin_weights=MC.lin_state_dict(MC.synthetic_lins()))
        lp_key = "lpips_synthetic"

    frames = {}
    for mode in ("fp16x3", "fp16f8", "fp16"):
        net.set_precision(mode)
        imitator.personalize("", src_smpl=src_theta.numpy(), src_img=src_img)       # source features in this mode too
        enc, res = imitator.src_info["feats"]
        imitator.first_cam = sets[0][0:1, 0:3].to(dev)
        out = []
        for th in sets:
            det = body.get_details(imitator.swap_smpl(imitator.src_info["cam"], imitator.src_info["shape"], th.to(dev), "smooth"))
            c = render.correspond(det["cam"].contiguous(), det["verts"].contiguous(), imitator.src_info["p2verts"],
                                  imitator.src_info["img"])
            out.append(net.inference(enc, res, c["tsf_inputs"], c["T"], bg=imitator.src_info["bg"])[2].clone())
        frames[mode] = torch.cat(out)
    ref = frames["fp16x3"]
    name, power = card()
    line = dict(card=name, power_limit=power, size=size, frames=int(ref.shape[0]), against="fp16x3")
    for mode in ("fp16f8", "fp16"):
        sc = M.score_frames(frames[mode], ref, lpips=lp)
        fin = torch.isfinite(sc["psnr"])
        line[mode] = dict(
            max_abs=float((frames[mode] - ref).abs().max()),
            ssim_mean=float(sc["ssim"].mean()), ssim_min=float(sc["ssim"].min()),
            psnr_mean_db=float(sc["psnr"][fin].mean()) if bool(fin.any()) else float("inf"),
            psnr_min_db=float(sc["psnr"].min()),
            **{lp_key + "_mean": float(sc["lpips"].double().mean()), lp_key + "_max": float(sc["lpips"].max())})
    print(json.dumps(line))


if __name__ == "__main__":
    main()
