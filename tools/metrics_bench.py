"""Frames per second of the paired metrics on the GPU (impersonator_b200.metrics) next to the CPU oracle.

    python tools/metrics_bench.py [--batch 32] [--iters 20]

For 256 and 512 px frame pairs: SSIM + PSNR (one lwb_ssim_psnr call) and LPIPS (AlexNet on the conv engine + the tap
kernels, synthetic weights: the speed does not depend on the values), timed with CUDA events over ``--iters`` calls
after warm-up, inputs already on the device.  The CPU column is oracle/metrics_ref.py (float64 numpy / torch, the
restatement of skimage and PNetLin the tests use) on a few frames of the same host.  Prints one JSON line with the card
name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

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
        line["%d" % size] = dict(gpu_ssim_psnr_fps=round(gpu_ssim, 1), gpu_lpips_fps=round(gpu_lpips, 1),
                                 cpu_ssim_psnr_fps=round(cpu_ssim, 2), cpu_lpips_fp32_fps=round(cpu_lpips, 2))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
