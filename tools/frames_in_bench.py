"""Input path: decoded uint8 frames -> the Imitator's generator input (S x S) and HMR input (224 x 224), per frame at
batch 16, through the reference's host route after cv2.imread and through lwb_frames_in, which the Imitator uses.

  host    the reference's computation: cvtColor + cv2.resize to S + cv2.resize to 224 + float conversion
          (x / 255 * 2 - 1) + H2D of both
  device  pinned uint8 H2D of the frames + one lwb_frames_in launch
  kernel  lwb_frames_in alone (CUDA events over many launches), with the bytes it must move (each source byte read once,
          both float outputs written) over the kernel time, against the H100 SXM data-sheet HBM3 peak of 3.35 TB/s

Both routes end in a device synchronise; they are timed with a host clock, alternating, median of the repeats.  Prints
the card's name and power limit, read in the same run, and one JSON line.  Usage: python tools/frames_in_bench.py"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from impersonator_b200 import _lib, kernels as K  # noqa: E402

HBM_PEAK = 3.35e12


def card():
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        power = out.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def host_route(frames, size, dev):
    import cv2
    img, hmr = [], []
    for f in frames:
        rgb = cv2.cvtColor(f, cv2.COLOR_BGR2RGB)
        img.append((cv2.resize(rgb, (size, size)).astype(np.float32) / 255.0).transpose((2, 0, 1)) * 2 - 1.0)
        hmr.append(cv2.resize(rgb, (224, 224)).astype(np.float32).transpose((2, 0, 1)) / 255.0 * 2 - 1.0)
    a = torch.from_numpy(np.stack(img)).to(dev)
    b = torch.from_numpy(np.stack(hmr)).to(dev)
    torch.cuda.synchronize()
    return a, b


def device_route(frames, size):
    img, hmr, _ = K.frames_in(frames, size, want_img=True, want_hmr=True)
    torch.cuda.synchronize()
    return img, hmr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    _lib.require_gpu()
    dev = torch.device("cuda", torch.cuda.current_device())
    name, power = card()
    print("card: %s, power limit / max SM clock: %s" % (name, power))
    rng = np.random.default_rng(0)
    results = []
    for src in (256, 1024):
        n, S = args.batch, args.size
        frames = rng.integers(0, 256, (n, src, src, 3), dtype=np.uint8)
        # same outputs, same bits (the tests sweep this in full)
        a, b = host_route(frames, S, dev)
        c, d = device_route(frames, S)
        same = bool(torch.equal(a, c) and torch.equal(b, d))
        t_host, t_dev = [], []
        for _ in range(3):                                                   # warm-up
            host_route(frames, S, dev), device_route(frames, S)
        for _ in range(args.repeats):                                        # alternate the two routes
            t0 = time.perf_counter()
            host_route(frames, S, dev)
            t1 = time.perf_counter()
            device_route(frames, S)
            t2 = time.perf_counter()
            t_host.append(t1 - t0)
            t_dev.append(t2 - t1)
        on_dev = torch.from_numpy(frames).to(dev)
        img = torch.empty((n, 3, S, S), device=dev)
        hmr = torch.empty((n, 3, 224, 224), device=dev)
        launch = lambda: _lib.check(_lib.lib().lwb_frames_in(on_dev.data_ptr(), n, src, src, 1, S, img.data_ptr(), 224,
                                                             hmr.data_ptr(), None, _lib.stream()), "lwb_frames_in")
        for _ in range(10):
            launch()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.launches):
            launch()
        e1.record()
        torch.cuda.synchronize()
        k_s = e0.elapsed_time(e1) / 1e3 / args.launches
        nbytes = n * src * src * 3 + n * 3 * (S * S + 224 * 224) * 4
        r = dict(source=src, size=S, batch=n, bit_identical=same,
                 host_ms_per_frame=float(np.median(t_host)) * 1e3 / n, device_ms_per_frame=float(np.median(t_dev)) * 1e3 / n,
                 kernel_us_per_frame=k_s * 1e6 / n, kernel_bytes=nbytes, kernel_gbps=nbytes / k_s / 1e9,
                 kernel_share_of_hbm_peak=nbytes / k_s / HBM_PEAK)
        results.append(r)
        print("%4d^2 -> %d + 224, batch %d: host route %.3f ms/frame, device route %.3f ms/frame (%.1fx), kernel %.1f us/frame, "
              "%.0f GB/s = %.1f%% of 3.35 TB/s, bit-identical %s"
              % (src, S, n, r["host_ms_per_frame"], r["device_ms_per_frame"], r["host_ms_per_frame"] / r["device_ms_per_frame"],
                 r["kernel_us_per_frame"], r["kernel_gbps"], 100 * r["kernel_share_of_hbm_peak"], same))
    print(json.dumps(dict(card=name, power_limit=power, results=results)))


if __name__ == "__main__":
    main()
