"""Device time of the Mask R-CNN person detector per source image (impersonator_b200.detectors), with the conv
engine's share, on synthetic weights (the speed does not depend on the values).

    python tools/detector_bench.py [--size 256] [--iters 10]

Prints one JSON line: ms per source (CUDA events around ``PersonMaskRCNNDetector.inference``), the conv engine's
milliseconds inside it (CUDA events per plan launch, serialised) and the card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")[:2]]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    import torch
    from impersonator_b200 import _lib, detectors as D, kernels as K, synthetic as S
    _lib.require_gpu()
    torch.set_grad_enabled(False)
    det = D.PersonMaskRCNNDetector(ks=13, weights=S.synthetic_maskrcnn_state())
    img = S.synthetic_source(a.size)[0].cuda()
    for _ in range(2):
        det.inference(img)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        det.inference(img)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.iters
    K.profile_begin()
    det.inference(img)
    prof = K.profile_end()
    name, power = card()
    print(json.dumps({"detector_ms_per_source": round(ms, 3), "size": a.size,
                      "conv_ms_serialised": round(prof.get("conv", {}).get("ms", 0.0), 3),
                      "det_passes_ms_serialised": round(prof.get("det", {}).get("ms", 0.0), 3),
                      "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
