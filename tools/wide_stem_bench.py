"""Cost of the wide conditioning maps on the GPU: the 7x7 stem plan at 6, 14 and 18 input channels (8, 16 and 24 padded
channels: one, two and three K stages per filter row), and one ImpersonatorGenerator.inference step at batch 16 for the
generators of 'uv_seg' (6 input channels), 'par' (14) and 'binary' (18).

    python tools/wide_stem_bench.py [--batch 16] [--size 256] [--iters 50] [--repeats 3] [--out result.json]

Times come from CUDA events around ``iters`` back-to-back calls after a warm-up, the median of ``repeats`` windows; the
card's name, power limit and maximum SM clock are read in the same run and printed with the numbers.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from impersonator_b200 import _lib, kernels as K, synthetic as S          # noqa: E402
from impersonator_b200.generator import ImpersonatorGenerator, stem_cin_pad   # noqa: E402

WIDTHS = {"uv_seg": 6, "par": 14, "binary": 18}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn, iters, repeats):
    """Median ms per call over ``repeats`` windows of ``iters`` calls (after two warm-up calls)."""
    fn()
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / iters)
    return sorted(out)[len(out) // 2]


def stem_ms(dev, cin, B, size, iters, repeats):
    """The generator's stem plan (fp16x3 operands, the mode every precision runs it in)."""
    g = torch.Generator().manual_seed(cin)
    x = torch.randn(B, cin, size, size, generator=g).to(dev)
    w = (torch.randn(64, cin, 7, 7, generator=g) * 0.05).to(dev)
    c_pad = stem_cin_pad(cin)
    xs = K.nchw_to_nhwc_split(x, c_pad=c_pad, pad_hw=(3, 3, 3, 5), split=1)
    ws = K.pack_conv_weight_rowk(w, cpx=c_pad, split=1)
    d = K.make_conv_desc(B, size, size, c_pad, 64, 7, 7, stride=1, pad=3, split=1, rowk=True, row_pitch=size + 8)
    out = torch.empty((B, size, size, 64), dtype=torch.float32, device=dev)
    st = torch.zeros((B, 64, 2), dtype=torch.float64, device=dev)
    plan = K.ConvPlan(d, xs, None, ws, out, st)
    ms = timed(plan.run, iters, repeats)
    # the work the padded plan issues: 8 c_pad K per filter row, 7 rows, three fp16 products
    issued = 2.0 * B * size * size * 64 * 7 * 8 * c_pad * 3
    return dict(ms=ms, padded_channels=c_pad, k_stages=plan.launch_info()["k_stages"],
                issued_tflops=issued / ms / 1e9)


def step_ms(dev, cin, B, size, iters, repeats):
    """One ImpersonatorGenerator.inference call at batch B on shared source features (the Imitator's step)."""
    net = ImpersonatorGenerator(bg_dim=4, src_dim=cin, tsf_dim=cin, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    net = net.to(dev).eval()
    inp = S.synthetic_generator_inputs(B, size, seed=11, cin=cin)
    enc, res = net.encode_src(inp["src"].to(dev))
    tsf, T = inp["tsf"].to(dev), inp["T"].to(dev)
    bg = torch.zeros(1, 3, size, size, device=dev)
    return dict(ms=timed(lambda: net.inference(enc, res, tsf, T, bg=bg), iters, repeats))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    _lib.require_gpu()
    torch.set_grad_enabled(False)
    dev = torch.device("cuda:0")
    res = {"card": card(), "batch": a.batch, "size": a.size, "stem": {}, "step": {}}
    for name, cin in WIDTHS.items():
        res["stem"][cin] = stem_ms(dev, cin, a.batch, a.size, a.iters, a.repeats)
    for name, cin in WIDTHS.items():
        res["step"][name] = step_ms(dev, cin, a.batch, a.size, max(a.iters // 5, 5), a.repeats)
    base = res["step"]["uv_seg"]["ms"]
    for name in WIDTHS:
        res["step"][name]["vs_uv_seg"] = res["step"][name]["ms"] / base - 1.0
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as fp:
            json.dump(res, fp, indent=1)


if __name__ == "__main__":
    main()
