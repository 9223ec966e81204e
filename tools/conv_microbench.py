"""Micro-benchmark of single conv layers of the wgmma engine (CUDA events), run from the repository root on a GPU.

The layers are the ones the flagship step runs (256x256, 16 frames as two sub-batch streams of 8), each in the three
operand modes: fp16f8 (the default, split=2), fp16x3 (split=1) and single-pass fp16 (split=0).  The row-K stem has no
fp8 path and runs fp16x3 where fp16f8 is asked for, as in the generator.  Beside the time, every layer prints the
operand bytes per algorithmic FLOP that the TMA unit moves from L2 into shared memory: for a schedule that fetches a
16-row activation tile per filter tap ("tap"), for y-halo tap groups on 16 x 8 tiles ("grp16"), and for the tiles the
engine runs ("run"): the same 16 x 8 tiles for N tiles of 16..128, the swapped 32 x 8 tiles for an N tile of 64.

    python tools/conv_microbench.py [--batch 8] [--reps 50] [--only res] [--json out.json]

``--compare A B`` times the builds of two source trees (each a checkout with its library built) against each other:
one worker process per tree, both on the same GPU, the same layer and mode timed in both, ``--rounds`` times with the
order alternating, and the median of each printed with their ratio B / A.

    python tools/conv_microbench.py --compare ../parent . [--batch 8] [--rounds 7] [--json cmp.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

K = merge_transposed_weight = None


def load(tree):
    """Imports the conv engine of the source tree at `tree`."""
    global K, merge_transposed_weight
    sys.path.insert(0, os.path.abspath(tree))
    from impersonator_b200 import kernels
    from impersonator_b200.binding import merge_transposed_weight as mtw
    K, merge_transposed_weight = kernels, mtw

TILE_H, TILE_W, KCHUNK, MAX_GROUP = 16, 8, 64, 8
SWAP_N_TILE, SWAP_TILE_H = 64, 32            # N = 64 plans run 64 channels x (32 x 8) pixels


def tile_rows(n_tile):
    return SWAP_TILE_H if n_tile == SWAP_N_TILE else TILE_H
MODES = (("fp16f8", 2), ("fp16x3", 1), ("fp16", 0))


def tap_groups(taps):
    """(view, dy, dx) per tap -> (groups, largest group): taps sharing view and dx with consecutive dy form one group
    (the rule of lwb_conv_plan_create)."""
    groups, run, prev = 0, 0, None
    longest = 0
    for v, dy, dx in sorted(taps, key=lambda t: (t[0], t[2], t[1])):
        if prev is not None and (v, dx) == (prev[0], prev[2]) and dy == prev[1] + 1 and run < MAX_GROUP:
            run += 1
        else:
            groups, run = groups + 1, 1
        longest = max(longest, run)
        prev = (v, dy, dx)
    return groups, longest


def launch_taps(spec):
    """Per launch of the plan: the (view, dy, dx) list of its taps."""
    kind, k = spec["kind"], spec.get("k", 3)
    if kind == "rowk":
        return [[(0, ky, 0) for ky in range(7)]]
    if kind == "merged":
        return [[(0, t >> 1, t & 1) for t in range(4)]]
    if kind == "transposed":
        d = ([0], [0, 1])
        return [[(0, dy, dx) for dy in d[a] for dx in d[b]] for a in range(2) for b in range(2)]
    kh, kw = (k, 1) if kind == "heads" else (k, k)
    pad, pad_w = k // 2, (0 if kind == "heads" else k // 2)
    taps = []
    for ky in range(kh):
        for kx in range(kw):
            oy, ox = ky - pad, kx - pad_w
            if spec.get("stride", 1) == 2:
                py, px = oy % 2, ox % 2
                taps.append((2 * py + px, (oy - py) // 2, (ox - px) // 2))
            else:
                taps.append((0, oy, ox))
    return [taps]


def operand_bytes(spec, n, n_tile, split, grouped, tile_h=TILE_H):
    """TMA bytes of the whole layer (activation hi/lo + weight hi/lo, every tile of tile_h x 8 pixels)."""
    ops = 2 if split else 1
    chunks = 1 if spec["kind"] == "rowk" else (spec["cin"] + spec.get("cin1", 0)) // KCHUNK
    dom = spec["h"] // 2 if spec.get("stride", 1) == 2 else spec["h"]
    ncols = 4 * spec["cout"] if spec["kind"] == "merged" else spec["cout"]
    tiles = n * -(-dom // tile_h) * -(-dom // TILE_W) * (ncols // n_tile)
    total = 0
    for taps in launch_taps(spec):
        if grouped:
            groups, longest = tap_groups(taps)
            a_rows = groups * (tile_h + longest - 1)
        else:
            a_rows = len(taps) * tile_h
        total += tiles * chunks * ops * (a_rows * TILE_W * 128 + len(taps) * n_tile * 128)
    return total


def make_plan(spec, n, split, dev):
    kind, h, cin, cout = spec["kind"], spec["h"], spec.get("cin", 8), spec["cout"]
    cin1 = spec.get("cin1", 0)
    x1 = None
    lo = lambda t: (t * 1e-3).half()                                # noqa: E731  (any bits: timing only)
    if kind == "rowk":
        split = min(split, 1)
        xs = torch.randn(n, h + 6, h + 8, 8, device=dev)
        x = (xs.half(), lo(xs))
        wt = torch.randn(cout, 6, 7, 7, device=dev) * 0.05
        w = K.pack_conv_weight_rowk(wt, split=split)
        d = K.make_conv_desc(n, h, h, 8, cout, 7, 7, stride=1, pad=3, split=split, rowk=True, row_pitch=h + 8)
        out_hw = h
    else:
        xs = torch.randn(n, h, h, cin, device=dev)
        x = (xs.half(), lo(xs))
        if cin1:
            x1s = torch.randn(n, h, h, cin1, device=dev)
            x1 = (x1s.half(), lo(x1s))
        k = spec.get("k", 3)
        if kind in ("transposed", "merged"):
            wt = torch.randn(cin, cout, 3, 3, device=dev) * 0.05
            if kind == "merged":
                w = K.pack_conv_weight(merge_transposed_weight(wt), split=split)
            else:
                w = K.pack_conv_weight(wt, transposed=True, split=split)
            d = K.make_conv_desc(n, h, h, cin, cout, 3, 3, stride=2, pad=1, transposed=True, split=split)
            if kind == "merged":
                d.transposed = 2
            out_hw = 2 * h
        elif kind == "heads":
            wt = torch.randn(cout, cin, k, 1, device=dev) * 0.05
            w = K.pack_conv_weight(wt, split=split)
            d = K.make_conv_desc(n, h, h, cin, cout, k, 1, pad=k // 2, pad_w=0, split=split, n_tile=spec["n_tile"])
            out_hw = h
        else:
            stride = spec.get("stride", 1)
            wt = torch.randn(cout, cin + cin1, k, k, device=dev) * 0.05
            w = K.pack_conv_weight(wt, split=split)
            d = K.make_conv_desc(n, h, h, cin, cout, k, k, stride=stride, pad=k // 2, cin1=cin1, split=split)
            out_hw = d.h_out
    out = torch.empty((n, out_hw, out_hw, cout), device=dev)
    st = torch.zeros((n, cout, 2), dtype=torch.float64, device=dev)
    return K.ConvPlan(d, x, x1, w, out, st), split


# the flagship's conv layers per sub-batch stream (ImpersonatorGenerator, 256x256, repeat_num 6, n_down 3)
LAYERS = [
    ("stem R7x7 8->64 @256", dict(kind="rowk", h=256, cout=64)),
    ("enc C3x3s2 64->128 @256", dict(kind="conv", stride=2, h=256, cin=64, cout=128)),
    ("enc C3x3s2 128->256 @128", dict(kind="conv", stride=2, h=128, cin=128, cout=256)),
    ("enc C3x3s2 256->512 @64", dict(kind="conv", stride=2, h=64, cin=256, cout=512)),
    ("res C3x3 512->512 @32 (x12)", dict(kind="conv", h=32, cin=512, cout=512)),
    ("dec T3x3 512->256 @32 (4 phases)", dict(kind="transposed", h=32, cin=512, cout=256)),
    ("skip C3x3 256+256->256 @64", dict(kind="conv", h=64, cin=256, cin1=256, cout=256)),
    ("dec T3x3 256->128 @64 (merged)", dict(kind="merged", h=64, cin=256, cout=128)),
    ("skip C3x3 128+128->128 @128", dict(kind="conv", h=128, cin=128, cin1=128, cout=128)),
    ("dec T3x3 128->64 @128 (merged)", dict(kind="merged", h=128, cin=128, cout=64)),
    ("skip C3x3 64+64->64 @256", dict(kind="conv", h=256, cin=64, cin1=64, cout=64)),
    ("heads C7x1 64->28 @256 (N 32)", dict(kind="heads", k=7, h=256, cin=64, cout=32, n_tile=32)),
]


def time_plan(plan, reps):
    for _ in range(3):
        plan.run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        plan.run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def worker(tree, batch, reps):
    """--compare worker: one request per line on stdin, "<layer index> <split>", answered with the time in ms."""
    load(tree)
    dev = torch.device("cuda")
    torch.set_grad_enabled(False)
    for req in sys.stdin:
        li, split = map(int, req.split())
        torch.manual_seed(0)
        plan, _ = make_plan(LAYERS[li][1], batch, split, dev)
        print(repr(time_plan(plan, reps)), flush=True)
        del plan


def compare(a):
    trees = a.compare
    cmd = [sys.executable, os.path.abspath(__file__), "--batch", str(a.batch), "--reps", str(a.reps), "--worker"]
    procs = [subprocess.Popen(cmd + [t], stdin=subprocess.PIPE, stdout=subprocess.PIPE, text=True) for t in trees]

    def ask(p, li, split):
        p.stdin.write("%d %d\n" % (li, split))
        p.stdin.flush()
        return float(p.stdout.readline())

    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("A = %s, B = %s; %s; batch %d, %d rounds x %d reps" % (trees[0], trees[1], gpu, a.batch, a.rounds, a.reps))
    print("%-34s %-7s %9s %9s %7s" % ("layer", "mode", "A ms", "B ms", "B / A"))
    rows = []
    for li, (name, _) in enumerate(LAYERS):
        if a.only and a.only not in name:
            continue
        for mode, split in MODES:
            ms = ([], [])
            for r in range(a.rounds):
                for i in ((0, 1) if r % 2 == 0 else (1, 0)):
                    ms[i].append(ask(procs[i], li, split))
            med = [statistics.median(m) for m in ms]
            rows.append(dict(layer=name, mode=mode, a_ms=med[0], b_ms=med[1], ratio=med[1] / med[0], a_all=ms[0], b_all=ms[1]))
            print("%-34s %-7s %9.4f %9.4f %7.3f" % (name, mode, med[0], med[1], med[1] / med[0]), flush=True)
    for p in procs:
        p.stdin.close()
        p.wait()
    tot = [sum(r[k] for r in rows if r["mode"] == "fp16f8") for k in ("a_ms", "b_ms")]
    print("fp16f8 total: A %.4f ms, B %.4f ms, B / A %.3f" % (tot[0], tot[1], tot[1] / tot[0]))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(gpu=gpu, a=trees[0], b=trees[1], batch=a.batch, reps=a.reps, rounds=a.rounds, rows=rows), f, indent=1)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--only", default="", help="substring filter on the layer name")
    ap.add_argument("--json", default="", help="also write the rows to this file")
    ap.add_argument("--compare", nargs=2, metavar=("A", "B"), help="time the builds of two source trees against each other")
    ap.add_argument("--rounds", type=int, default=7, help="--compare: timings per layer, mode and tree")
    ap.add_argument("--worker", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.worker, a.batch, a.reps)
    if a.compare:
        return compare(a)
    load(".")
    dev = torch.device("cuda")
    torch.manual_seed(0)
    torch.set_grad_enabled(False)
    rows = []
    print("%-34s %-7s %9s %9s %10s %10s %10s" % ("layer (batch %d)" % a.batch, "mode", "ms", "TFLOP/s", "B/FLOP tap",
                                                  "B/FLOP g16", "B/FLOP run"))
    for name, spec in LAYERS:
        if a.only and a.only not in name:
            continue
        for mode, split in MODES:
            plan, ran = make_plan(spec, a.batch, split, dev)
            ms = time_plan(plan, a.reps)
            n_tile = spec.get("n_tile") or (128 if (4 * spec["cout"] if spec["kind"] == "merged" else spec["cout"]) % 128 == 0 else 64)
            bpf = [operand_bytes(spec, a.batch, n_tile, ran, g) / plan.flops for g in (False, True)]
            bpf.append(operand_bytes(spec, a.batch, n_tile, ran, True, tile_rows(n_tile)) / plan.flops)
            row = dict(layer=name, mode=mode, ran_split=ran, ms=ms, tflops=plan.flops / ms / 1e9, n_tile=n_tile,
                       tile_h=tile_rows(n_tile), bytes_per_flop_per_tap=bpf[0], bytes_per_flop_grouped=bpf[1],
                       bytes_per_flop_run=bpf[2])
            rows.append(row)
            print("%-34s %-7s %9.4f %9.1f %10.4f %10.4f %10.4f" % (name, mode + ("*" if ran != split else ""), ms, row["tflops"],
                                                                  bpf[0], bpf[1], bpf[2]))
            del plan
    print("* the row-K stem has no fp8 path: fp16x3 operands")
    props = torch.cuda.get_device_properties(0)
    print("device: %s" % props.name)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(device=props.name, batch=a.batch, reps=a.reps, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
