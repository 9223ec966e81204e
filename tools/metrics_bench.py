"""Frames per second of the paired metrics on the GPU (impersonator_b200.metrics) next to the CPU oracle.

    python tools/metrics_bench.py [--batch 32] [--iters 20]

For 256 and 512 px frame pairs: SSIM + PSNR (one lwb_ssim_psnr call) and LPIPS (AlexNet on the conv engine + the tap
kernels, synthetic weights: the speed does not depend on the values) and the InceptionV3 features of IS / FID (the
conv engine in fp16x3, next to torchvision's Inception3 in fp32 on cuDNN with TF32 off), timed with CUDA events over
``--iters`` calls after warm-up, inputs already on the device; then the device Frechet distance of two 4096 x 2048
float64 feature sets.  The CPU column is oracle/metrics_ref.py (float64 numpy / torch, the
restatement of skimage and PNetLin the tests use) on a few frames of the same host.  Prints one JSON line with the card
name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu_frames", type=int, default=2)
    args = ap.parse_args()

    import torch
    import metrics_cases as MC
    from detector_bench import card
    from impersonator_b200 import _lib, metrics as M
    from oracle import metrics_ref as R

    _lib.require_gpu()
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    lp = M.LPIPS(dev, weights=MC.alexnet_state_dict(convs), lin_weights=MC.lin_state_dict(lins))
    # InceptionV3 features (IS / FID) on the conv engine, and torchvision's Inception3 up to the same 2048 pool features
    # in fp32 on cuDNN with TF32 off, both on the metric classes' preprocess; synthetic weights (calibrated BN statistics)
    import inception_cases as IC
    import torch.nn.functional as F
    import torchvision
    gold = np.load(os.path.join(ROOT, "tests", "golden", "inception.npz"))
    sd = IC.golden_state_dict(gold)
    incep = M.InceptionFeatures(dev, weights=sd)
    tv = torchvision.models.inception_v3(weights=None, init_weights=False, aux_logits=True)
    tv.load_state_dict(sd, strict=False)
    tv = tv.to(dev).eval()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    names = ["Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "maxpool1", "Conv2d_3b_1x1", "Conv2d_4a_3x3", "maxpool2",
             "Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e", "Mixed_7a",
             "Mixed_7b", "Mixed_7c", "avgpool"]

    def tv_features(x):
        y = F.interpolate(x * 2 - 1, size=(299, 299), mode='bilinear', align_corners=False)
        for nm in names:
            y = getattr(tv, nm)(y)
        return y[:, :, 0, 0]

    g = torch.Generator(device=dev).manual_seed(0)
    name, power = card()
    line = dict(card=name, power_limit=power, batch=args.batch, cpu_threads=torch.get_num_threads())
    for size in (256, 512):
        p = torch.rand((args.batch, 3, size, size), device=dev, generator=g)
        t = torch.rand((args.batch, 3, size, size), device=dev, generator=g)

        def timed(fn):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            torch.cuda.synchronize()
            return args.batch * args.iters / (e0.elapsed_time(e1) / 1e3)

        gpu_ssim = timed(lambda: M.ssim_psnr(p, t))
        gpu_lpips = timed(lambda: lp(p, t))
        k = args.cpu_frames
        ph, th = p[:k].cpu().numpy(), t[:k].cpu().numpy()
        t0 = time.time()
        R.ssim_scores(ph, th)
        R.psnr_scores(ph, th)
        cpu_ssim = k / (time.time() - t0)
        t0 = time.time()
        R.lpips(torch.from_numpy(th) * 2 - 1, torch.from_numpy(ph) * 2 - 1, convs, lins, dtype=torch.float32)
        cpu_lpips = k / (time.time() - t0)
        gpu_incep = timed(lambda: incep(p))
        tv_incep = timed(lambda: tv_features(p))
        line["%d" % size] = dict(gpu_ssim_psnr_fps=round(gpu_ssim, 1), gpu_lpips_fps=round(gpu_lpips, 1),
                                 cpu_ssim_psnr_fps=round(cpu_ssim, 2), cpu_lpips_fp32_fps=round(cpu_lpips, 2),
                                 gpu_inception_fps=round(gpu_incep, 1), torchvision_inception_fp32_fps=round(tv_incep, 1))
    a = torch.rand((4096, 2048), device=dev, generator=g, dtype=torch.float64)
    b = torch.rand((4096, 2048), device=dev, generator=g, dtype=torch.float64)
    M.FIDMetric.fid_score_func(a, b)
    torch.cuda.synchronize()
    t0 = time.time()
    for _ in range(3):
        M.FIDMetric.fid_score_func(a, b)                               # returns a float: ends in a device sync
    line["frechet_d2048_s"] = round((time.time() - t0) / 3, 3)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
