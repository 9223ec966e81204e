"""How much of the HBM-bound work of one sub-batch stream runs under the other stream's convolutions (run on a GPU).

Runs the bench workload (16 frames at 256 x 256, default mode: fp16f8, captured step graph, two sub-batch streams of 8)
and takes one torch.profiler trace with CUDA activities of a few replayed steps (OUT/trace.pt.trace.json; OUT defaults
to a new temporary directory).
From the trace it reports, per stream and kernel class, the busy time per step and how much of it overlaps a k_conv_wg
running on another stream; the step time comes from CUDA events over replays without the profiler, the card name and
power limit from nvidia-smi in the same run.  Then, per kernel instance the generator launches: registers, static and
dynamic shared memory, blocks per SM alone (occupancy API) and beside one resident CTA of each conv instance
(kernels.blocks_beside).

    python tools/stream_overlap.py [--out DIR] [--root DIR] [--steps 5] [--json FILE]

--root imports the package from another checkout (e.g. the parent commit's build) so that two builds are compared
with the same script; the resource table needs lwb_conv_kernel_resources and is skipped where the library lacks it.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

CLASSES = (("k_conv_wg", "conv"), ("k_norm_act", "norm"), ("k_finalize_stats", "finalize"), ("k_heads", "heads"),
           ("k_nchw_to_nhwc_split", "input"))


def kernel_class(name):
    for key, cls in CLASSES:
        if key in name:
            return cls
    return "other"


def union(iv):
    out = []
    for a, b in sorted(iv):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def overlap(a, b, c, d):
    return max(0.0, min(b, d) - max(a, c))


def analyse(trace_path, steps):
    """-> {stream: {class: {"n", "busy_ms", "under_conv_ms"}}} per step, from the kernel events of a chrome trace."""
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    kern = [e for e in events if e.get("cat") == "kernel" and "dur" in e]
    by_stream = {}
    for e in kern:
        st = e.get("args", {}).get("stream", -1)
        by_stream.setdefault(st, []).append((kernel_class(e["name"]), float(e["ts"]), float(e["ts"]) + float(e["dur"])))
    conv_of = {st: union([(a, b) for c, a, b in ks if c == "conv"]) for st, ks in by_stream.items()}
    report = {}
    for st, ks in by_stream.items():
        others = union([iv for o, ivs in conv_of.items() if o != st for iv in ivs])
        rows = {}
        for cls, a, b in ks:
            r = rows.setdefault(cls, {"n": 0, "busy_ms": 0.0, "under_conv_ms": 0.0})
            r["n"] += 1
            r["busy_ms"] += (b - a) / 1e3
            r["under_conv_ms"] += sum(overlap(a, b, c, d) for c, d in others) / 1e3
        for r in rows.values():
            r["n"] /= steps
            r["busy_ms"] /= steps
            r["under_conv_ms"] /= steps
        report[str(st)] = rows
    return report


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def resources(K, torch):
    if not hasattr(K, "conv_kernel_resources"):
        return None
    props = torch.cuda.get_device_properties(0)
    convs = {"k_conv_wg<%d,%d>" % nm: K.conv_kernel_resources(*nm) for nm in K.GENERATOR_CONV_INSTANCES}
    rows = []
    for name, r in convs.items():
        rows.append(dict(kernel=name, **r))
    for name, (which, c) in K.GENERATOR_GLUE_INSTANCES.items():
        r = K.glue_kernel_resources(which, c)
        rows.append(dict(kernel=name, beside={cn: K.blocks_beside(cr, r, props) for cn, cr in convs.items()}, **r))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--json")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from torch.profiler import ProfilerActivity, profile
    from impersonator_b200 import _lib, kernels as K, synthetic as S
    from impersonator_b200.generator import ImpersonatorGenerator
    from impersonator_b200.graph import CapturedStep
    from impersonator_b200.hmr import HumanModelRecovery
    from impersonator_b200.imitator import Imitator
    from impersonator_b200.nmr import SMPLRenderer

    _lib.require_gpu()
    torch.set_grad_enabled(False)
    dev = torch.device("cuda", 0)
    B, size = 16, 256
    # the bench.py workload: synthetic weights (seed 0), one personalized source, 16 target frames per step
    v, f = S.uv_sphere()
    tabs = S.synthetic_tables()
    net = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6)
    net.load_state_dict(S.fill_state_dict(net.state_dict(), seed=0))
    net = net.to(dev).eval()
    src_img = S.synthetic_source(size)
    render = SMPLRenderer(image_size=size, faces=f.numpy(), map_fn=tabs["map_fn"], has_front=False).to(dev)

    class Opt(object):
        image_size, batch_size, bg_model, repeat_num, cond_nc = size, B, "ORIGINAL", 6, 3
        bg_ks, ft_ks, front_warp, only_vis = 13, 3, False, False
    body = HumanModelRecovery(smpl_model=S.synthetic_smpl_model(seed=3)).to(dev)
    imitator = Imitator(Opt(), generator=net, hmr=body, render=render, device=dev)
    src_theta = S.synthetic_smpl_params(1, seed=5)[0]
    imitator.personalize("", src_smpl=src_theta.numpy(), src_img=src_img)
    th = S.synthetic_smpl_params(B, seed=1000)
    imitator.first_cam = th[0:1, 0:3].to(dev)
    det = body.get_details(imitator.swap_smpl(imitator.src_info["cam"], imitator.src_info["shape"], th.to(dev), "smooth"))
    cam, verts = det["cam"].contiguous(), det["verts"].contiguous()
    enc, res = imitator.src_info["feats"]
    bg = imitator.src_info["bg"]
    p2v, simg = imitator.src_info["p2verts"], imitator.src_info["img"]

    def step_body(cam, verts):
        out = render.correspond(cam, verts, p2v, simg)
        return net.inference(enc, res, out["tsf_inputs"], out["T"], bg=bg)[2]

    step = CapturedStep(step_body, dict(cam=cam, verts=verts))
    for _ in range(10):
        step(cam=cam, verts=verts)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n_timed = 100
    e0.record()
    for _ in range(n_timed):
        step(cam=cam, verts=verts)
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / n_timed

    out_dir = args.out or tempfile.mkdtemp(prefix="stream_overlap_")
    os.makedirs(out_dir, exist_ok=True)
    trace = os.path.join(out_dir, "trace.pt.trace.json")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step(cam=cam, verts=verts)
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)

    result = {"card": card(), "root": os.path.abspath(args.root), "graph": bool(step.captured), "trace": trace,
              "step_ms": step_ms, "frames_per_s": B / step_ms * 1e3,
              "streams": analyse(trace, args.steps), "resources": resources(K, torch)}
    print("card: %s   step %.3f ms (%.0f frames/s), graph %s" % (result["card"], step_ms, result["frames_per_s"],
                                                                result["graph"]))
    print("%-8s %-9s %7s %9s %14s %6s" % ("stream", "class", "n/step", "busy ms", "under conv ms", "share"))
    tot = {}
    for st, rows in sorted(result["streams"].items()):
        for cls, r in sorted(rows.items()):
            share = r["under_conv_ms"] / r["busy_ms"] if r["busy_ms"] else 0.0
            print("%-8s %-9s %7.1f %9.3f %14.3f %6.2f" % (st, cls, r["n"], r["busy_ms"], r["under_conv_ms"], share))
            t = tot.setdefault(cls, [0.0, 0.0])
            t[0] += r["busy_ms"]
            t[1] += r["under_conv_ms"]
    for cls, (b, u) in sorted(tot.items()):
        print("all      %-9s %7s %9.3f %14.3f %6.2f" % (cls, "", b, u, u / b if b else 0.0))
    if result["resources"] is None:
        print("resources: this build has no lwb_conv_kernel_resources")
    else:
        convs = [r["kernel"] for r in result["resources"] if "beside" not in r]
        print("%-24s %5s %7s %7s %6s %6s  blocks/SM beside one CTA of %s" %
              ("kernel", "regs", "static", "dynamic", "local", "alone", ", ".join(convs)))
        for r in result["resources"]:
            beside = " ".join("%d" % r["beside"][c] for c in convs) if "beside" in r else \
                "(launch regs; consumers %d after setmaxnreg, %d threads)" % (r["consumer_regs"], r["threads"])
            print("%-24s %5d %7d %7d %6d %6d  %s" % (r["kernel"], r["regs"], r["static_smem"], r["dyn_smem"],
                                                   r["local_bytes"], r["blocks_alone"], beside))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
