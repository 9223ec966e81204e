"""The census of conv-engine plans the networks bind, and the windowed float64 check that test_conv_census_gpu.py runs on
each of them.  Helper module for the conv tests, not a test file.

``collect(config, mode)`` builds one network stream on the CPU (the kernel front-ends replaced by the stand-ins of
tests/kernel_emulator.py, LWB_PRECISION set to ``mode``) and records every convolution at ``PlanBinder.finalize``, before
packing: the lwb_conv_desc fields (all but w_exp, which packing sets), the weight shape (already merged for merged
transposed convs), cout_pad / cin_pad, the operand shapes and whether InstanceNorm statistics are bound.  Nothing is packed
or computed.  Every network binds its convolutions through PlanBinder, so the census sees all of them.

``CENSUS`` is the committed table of distinct plans over ``CONFIGS`` (the production configurations); each entry names the
(config, layer index) bindings, so a failure names the real layer, and the operand modes it runs in.
test_conv_census_cpu.py keeps it equal to the live census.

Out of scope: split 0 (the single-pass fp16 mode is not parity-gated) and the developer switches LWB_HALO,
LWB_CONVT_MERGE=0 and LWB_TC_HEADS=0.  The halo, per-phase transposed and CUDA-core heads paths they select are covered by
test_conv_gpu.py and test_conv_emulation_gpu.py.

The windowed check.  Emulating whole production layers in float64 on the CPU would take hours, so each case is checked on
windows of whole tiles of its plan's orientation (16 x 8 output pixels, 32 x 8 for the N = 64 tiles; the input-grid tile
mapped to the output for transposed convs), with all cout_pad channels: the first and the last tile of the first and the
last image (the last ones partial where the domain is), the first tile of the last tile row, and six seeded-random tiles.
Where one image costs at most ``IMAGE_BUDGET`` multiply-adds x 2 per product, the first and the last whole image are
checked instead.  ``conv_emulation.emulate`` splits x and w elementwise before it calls the conv, so emulating a crop with
a valid (padding 0) conv is exact.
"""
import collections
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import kernel_emulator
from conv_emulation import emulate

SMS = 132                        # H100 SXM
TILE_H, TILE_W, SWAP_N_TILE, SWAP_TILE_H, MAX_N_TILE = 16, 8, 64, 32, 128      # csrc/conv_tc.cu
# EMU_BAR (conv_emulation) holds for reductions up to 3x3 x 512 channels.  The kernel's fp32 accumulators add one MMA
# step after another, so their rounding error grows with the reduction length K: on an H100 the fp16x3 error against the
# emulation was 0.70 of EMU_BAR at K = 4608 and 1.53 at K = 12544 (the box head's FC6), while staying at 0.23 of the fp32
# bar.  Longer reductions are held to EMU_BAR x K / EMU_K.
EMU_K = 4608
IMAGE_BUDGET = 2e9               # FLOP (2 x MACs) of one product over one image, above which windows are checked
N_RANDOM = 6

MODES = {"fp16f8": 2, "fp16x3": 1}
DESC_FIELDS = ("n", "h_in", "w_in", "h_out", "w_out", "cin0", "cin1", "cout", "kh", "kw", "stride", "pad", "dil",
               "transposed", "split", "rowk", "row_pitch", "n_tile", "halo", "pad_w")
CPU = torch.device("cpu")


# ------------------------------------------------------------------------------------------------------------- configs
def _generator():
    from impersonator_b200.generator import ImpersonatorGenerator
    return ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6).eval()


def _unet(B, size, which="tsf_model"):
    def build(split):
        from impersonator_b200.generator import _Stream
        return _Stream(getattr(_generator(), which), B, size, size, CPU, split)
    return build


def _hmr(B):
    def build(split):
        from impersonator_b200 import synthetic as S
        from impersonator_b200.hmr import HumanModelRecovery, _HmrStream
        return _HmrStream(HumanModelRecovery(smpl_model=S.synthetic_smpl_model(seed=3)).eval(), B, CPU, split)
    return build


def _inpaintor(split):
    from impersonator_b200.inpaintor import InpaintSANet, _InpaintStream
    return _InpaintStream(InpaintSANet(c_dim=4).eval(), 1, 256, 256, CPU, split)


def _detector(size):
    def build(split):
        from impersonator_b200.detectors import MaskRCNN, _DetStream
        return _DetStream(MaskRCNN(), size, size, CPU)
    return build


def _lpips(split):
    import metrics_cases as MC
    from impersonator_b200 import metrics as M
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    return M._AlexStream(M.LPIPS(weights=MC.alexnet_state_dict(convs), lin_weights=MC.lin_state_dict(lins)), 32, 256, 256,
                         CPU)


def _inception(split):
    import inception_cases as IC
    from impersonator_b200 import metrics as M
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inception.npz"))
    return M.InceptionFeatures(weights=IC.golden_state_dict(gold)).stream(32, 256, 256)


BOTH, FP16X3 = ("fp16f8", "fp16x3"), ("fp16x3",)
# name -> (builder(split), operand modes it runs in)
CONFIGS = collections.OrderedDict([
    # bench.py's batch 16 at 256, split by generator._sub_batches into two sub-batch streams of 8
    ("unet_b8_256", (_unet(8, 256), BOTH)),
    # the same batch where sub-batching does not apply (per-frame sources, LWB_STREAMS=1)
    ("unet_b16_256", (_unet(16, 256), BOTH)),
    # test_configs_gpu config 5: batch 8 at 512, two sub-batches of 4
    ("unet_b4_512", (_unet(4, 512), BOTH)),
    # ImpersonatorGenerator.encode_src / infer_front: the source image through src_model
    ("src_b1_256", (_unet(1, 256, "src_model"), BOTH)),
    # the BG net on the one source background (Imitator.personalize)
    ("bg_b1_256", (_unet(1, 256, "bg_model"), BOTH)),
    # HMR on one image (personalize) and on a chunk of opt.batch_size target frames (imitator.py chunk_smpls, bench 16)
    ("hmr_b1", (_hmr(1), BOTH)),
    ("hmr_b16", (_hmr(16), BOTH)),
    # the DeepFill-v2 background inpaintor on one 256 source (bench.py, opt.bg_model != 'ORIGINAL')
    ("inpaintor_b1_256", (_inpaintor, BOTH)),
    # the Mask R-CNN person detector pins fp16x3; both sizes resize to 800 x 800
    ("detector_256", (_detector(256), FP16X3)),
    ("detector_512", (_detector(512), FP16X3)),
    # LPIPS and Inception pin fp16x3; the metric classes' calculate_score batch is 32 frames (LPIPS: 64 images)
    ("lpips_b32_256", (_lpips, FP16X3)),
    ("inception_b32_256", (_inception, FP16X3)),
])


# ------------------------------------------------------------------------------------------------------------- collect
Binding = collections.namedtuple("Binding", "desc weight cout_pad cin_pad x x1 stats")


class _NoRun(object):
    def __init__(self, desc):
        self.desc = desc

    def run(self):
        raise AssertionError("the census builds streams only")


def collect(config, mode):
    """[(layer index, Binding)] of one config in one operand mode, in binding order."""
    from impersonator_b200 import binding, metrics as M
    build, _ = CONFIGS[config]
    rec = []

    def finalize(self):
        convs, self._convs = self._convs, []
        for r in convs:
            rec.append(Binding(tuple(getattr(r.desc, f) for f in DESC_FIELDS), tuple(r.weight.shape), r.cout_pad,
                               r.cin_pad, tuple(r.x[0].shape), tuple(r.x1[0].shape) if r.x1 is not None else None,
                               r.stats is not None))
            r.plan = _NoRun(r.desc)
            r.weight = None

    with pytest.MonkeyPatch.context() as mp, torch.no_grad():
        kernel_emulator.install(mp)
        mp.setenv("LWB_PRECISION", mode)
        for var in ("LWB_HALO", "LWB_CONVT_MERGE", "LWB_TC_HEADS"):
            mp.delenv(var, raising=False)
        mp.setattr(M, "_device", lambda device: CPU)
        mp.setattr(binding.PlanBinder, "finalize", finalize)
        build(binding.split_mode())
    return list(enumerate(rec))


def key_of(b):
    """A plan without its operand mode: the descriptor with split zeroed, and the binding's shapes."""
    d = dict(zip(DESC_FIELDS, b.desc))
    d["split"] = 0
    return (tuple(d[f] for f in DESC_FIELDS), b.weight, b.cout_pad, b.cin_pad, b.x, b.x1, b.stats)


def live_census(configs=None):
    """{plan key: {"splits": set, "uses": [(config, layer)]}} over the given configs in all their modes."""
    out = collections.OrderedDict()
    for name in configs or CONFIGS:
        for mode in CONFIGS[name][1]:
            for layer, b in collect(name, mode):
                e = out.setdefault(key_of(b), {"splits": set(), "uses": []})
                e["splits"].add(dict(zip(DESC_FIELDS, b.desc))["split"])
                if (name, layer) not in e["uses"]:
                    e["uses"].append((name, layer))
    return out


# ------------------------------------------------------------------------------------------------------------ schedule
def n_tile_of(d):
    """The N tile and GEMM width lwb_conv_plan_create picks (pick_n_tile; 128 over 4 x cout for merged transposed)."""
    if d["transposed"] == 2:
        return MAX_N_TILE, 4 * d["cout"]
    f = d["n_tile"]
    if f > 0:
        return (MAX_N_TILE if f > MAX_N_TILE and f % MAX_N_TILE == 0 else f), d["cout"]
    for t in (128, 64, 32, 16):
        if d["cout"] % t == 0:
            return t, d["cout"]
    raise ValueError("no N tile divides cout %d" % d["cout"])


def schedule(d):
    """(n_tile, tile rows, tiles_y, tiles_x, N tiles, tiles per launch, tiles per CTA at SMS) of a plan."""
    nt, ncols = n_tile_of(d)
    th = SWAP_TILE_H if nt == SWAP_N_TILE else TILE_H
    dom_h, dom_w = (d["h_in"], d["w_in"]) if d["transposed"] else (d["h_out"], d["w_out"])
    ty, tx = -(-dom_h // th), -(-dom_w // TILE_W)
    total = d["n"] * ty * tx * (ncols // nt)
    return nt, th, ty, tx, ncols // nt, total, total / min(total, SMS)


# ----------------------------------------------------------------------------------------------------------- the table
Entry = collections.namedtuple("Entry", "name desc weight cout_pad cin_pad x x1 stats splits uses")


def entry_name(d, weight, x1):
    kind = "rowk" if d["rowk"] else ("convT" if d["transposed"] == 1 else ("convTm" if d["transposed"] == 2 else "conv"))
    cin = "%d+%d" % (d["cin0"], d["cin1"]) if d["cin1"] else "%d" % d["cin0"]
    s = "%s%dx%d_s%d_%s_%d_n%d_%dx%d" % (kind, d["kh"], d["kw"], d["stride"], cin, d["cout"], d["n"], d["h_out"], d["w_out"])
    if d["pad"] != d["kh"] // 2 and not d["transposed"]:
        s += "_p%d" % d["pad"]
    if d["pad_w"] >= 0:
        s += "_pw%d" % d["pad_w"]
    if d["dil"] != 1:
        s += "_d%d" % d["dil"]
    if d["n_tile"]:
        s += "_nt%d" % d["n_tile"]
    return s


def entries_of(census):
    out = []
    for (desc, weight, cout_pad, cin_pad, x, x1, stats), e in census.items():
        d = dict(zip(DESC_FIELDS, desc))
        out.append(Entry(entry_name(d, weight, x1), desc, weight, cout_pad, cin_pad, x, x1, stats,
                         tuple(sorted(e["splits"], reverse=True)), tuple(e["uses"])))
    names = collections.Counter(e.name for e in out)
    seen = collections.Counter()
    for i, e in enumerate(out):                     # the same shape bound with other padding / operands
        if names[e.name] > 1:
            seen[e.name] += 1
            out[i] = e._replace(name="%s_v%d" % (e.name, seen[e.name]))
    return out


def format_entry(e):
    d = dict(zip(DESC_FIELDS, e.desc))
    nt, th, ty, tx, nn, total, per = schedule(d)
    uses = ", ".join("(%r, %d)" % u for u in e.uses)
    return ("    # N tile %d, %dx%d tiles, %d x %d x %d N tiles x %d images = %d tiles, %.1f per CTA\n"
            "    Entry(%r, %r,\n          %r, %r, %r, %r, %r, %r, %r,\n          (%s,)),\n"
            % (nt, th, TILE_W, ty, tx, nn, d["n"], total, per, e.name, e.desc, e.weight, e.cout_pad, e.cin_pad, e.x, e.x1,
               e.stats, e.splits, uses))


def format_census(entries):
    return "CENSUS = [\n    # name, desc (DESC_FIELDS, split 0), weight shape, cout_pad, cin_pad, x, x1, stats, splits, (config, layer)\n" + \
        "".join(format_entry(e) for e in entries) + "]\n"


def label(e, split=None):
    """The entry and the layers that bind it, for assertion messages."""
    uses = ", ".join("%s#%d" % u for u in e.uses[:6]) + (" and %d more" % (len(e.uses) - 6) if len(e.uses) > 6 else "")
    return "%s%s [%s]" % (e.name, "" if split is None else " split %d" % split, uses)


# --------------------------------------------------------------------------------------------------- inputs and checks
GARBAGE = 1e3                    # finite, nonzero: the input channels between the layer's cin and cin_pad


def desc_of(e):
    return dict(zip(DESC_FIELDS, e.desc))


def real_dims(e):
    """(cin, cout, fp32 weight shape) of the layer itself: IOHW [cin, cout, 3, 3] for both transposed forms (the merged
    weight is built from it), OIHW otherwise; cin and cout without padding."""
    d = desc_of(e)
    if d["transposed"] == 2:
        return e.weight[1], e.weight[0] // 4, (e.weight[1], e.weight[0] // 4, 3, 3)
    if d["transposed"] == 1:
        return e.weight[0], e.weight[1], e.weight
    return e.weight[1], e.weight[0], e.weight


def make_inputs(e, seed):
    """Seeded N(0,1) NCHW input [n, cin0 + cin1, h_in, w_in] with GARBAGE in the channels from the layer's cin on, and
    weights N(0,1) / sqrt(fan-in) at the layer's real shape."""
    d = desc_of(e)
    cin, _, wshape = real_dims(e)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((d["n"], d["cin0"] + d["cin1"], d["h_in"], d["w_in"]), generator=g)
    x[:, cin:] = GARBAGE
    w = torch.randn(wshape, generator=g) / float(np.sqrt(cin * wshape[2] * wshape[3]))
    return x, w


def _crop(x, img, y0, y1, x0, x1):
    """x[img, :, y0:y1, x0:x1] as [1, C, y1 - y0, x1 - x0], zero outside the image."""
    c = torch.zeros((1, x.shape[1], y1 - y0, x1 - x0), dtype=x.dtype)
    sy0, sy1, sx0, sx1 = max(y0, 0), min(y1, x.shape[2]), max(x0, 0), min(x1, x.shape[3])
    if sy1 > sy0 and sx1 > sx0:
        c[:, :, sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = x[img:img + 1, :, sy0:sy1, sx0:sx1]
    return c


def window_conv(d, x, img, win):
    """(input crop, valid conv callable) whose result is output window ``win`` = (oy0, oy1, ox0, ox1) of image ``img``.
    x: NCHW input with the layer's cin channels (padded channels dropped)."""
    oy0, oy1, ox0, ox1 = win
    if d["transposed"]:                 # output rows 2i, 2i + 1 read input rows i, i + 1 (even window bounds)
        crop = _crop(x, img, oy0 // 2, oy1 // 2 + 1, ox0 // 2, ox1 // 2 + 1)
        return crop, lambda a, b: F.conv_transpose2d(a, b, stride=2, padding=1, output_padding=1)[:, :, :oy1 - oy0,
                                                                                                    :ox1 - ox0]
    s, dil = d["stride"], d["dil"]
    pw = d["pad_w"] if d["pad_w"] >= 0 else d["pad"]
    crop = _crop(x, img, oy0 * s - d["pad"], (oy1 - 1) * s - d["pad"] + dil * (d["kh"] - 1) + 1,
                 ox0 * s - pw, (ox1 - 1) * s - pw + dil * (d["kw"] - 1) + 1)
    return crop, lambda a, b: F.conv2d(a, b, stride=s, dilation=dil)


def image_flop(e):
    """2 x multiply-adds of one product over one image."""
    d = desc_of(e)
    cin, cout, wshape = real_dims(e)
    if d["transposed"]:
        return 2.0 * d["h_in"] * d["w_in"] * cin * cout * 9
    return 2.0 * d["h_out"] * d["w_out"] * cin * cout * wshape[2] * wshape[3]


def windows(e, seed=0):
    """[(image, (oy0, oy1, ox0, ox1))] the emulation checks: the first and the last image when one image is within
    IMAGE_BUDGET, else whole tiles of the plan's orientation (see the module docstring).  Every window spans all output
    channels, so it covers every N tile of its pixels."""
    d = desc_of(e)
    n = d["n"]
    if image_flop(e) <= IMAGE_BUDGET:
        return [(i, (0, d["h_out"], 0, d["w_out"])) for i in sorted({0, n - 1})]
    _, th, ty, tx, _, _, _ = schedule(d)
    dom_h, dom_w = (d["h_in"], d["w_in"]) if d["transposed"] else (d["h_out"], d["w_out"])
    f = 2 if d["transposed"] else 1
    picks = [(0, 0, 0), (0, ty - 1, tx - 1), (n - 1, 0, 0), (n - 1, ty - 1, tx - 1), (n - 1, ty - 1, 0)]
    rng = np.random.RandomState(seed)
    picks += [(int(rng.randint(n)), int(rng.randint(ty)), int(rng.randint(tx))) for _ in range(N_RANDOM)]
    out = []
    for img, y, x in picks:
        w = (img, (f * y * th, f * min((y + 1) * th, dom_h), f * x * TILE_W, f * min((x + 1) * TILE_W, dom_w)))
        if w not in out:
            out.append(w)
    return out


def reference(e, x, w, split, w_exp, img, win):
    """(float64 emulation of operand mode ``split``, fp32 conv) of one output window, [1, cout, h, w] on the CPU."""
    d = desc_of(e)
    cin = real_dims(e)[0]
    crop, conv = window_conv(d, x[:, :cin], img, win)
    return emulate(crop, w, conv, split, w_exp), conv(crop.float(), w.float())


def emulated_output(e, x, w, split, w_exp):
    """The whole NHWC float32 output the plan is meant to compute, from the emulation (the mutant tests' kernel)."""
    d = desc_of(e)
    ys = [reference(e, x, w, split, w_exp, i, (0, d["h_out"], 0, d["w_out"]))[0] for i in range(d["n"])]
    y = torch.cat(ys).float().permute(0, 2, 3, 1)
    return F.pad(y, (0, d["cout"] - y.shape[-1])).contiguous()


class CheckFailed(AssertionError):
    """A failed check of check_output; ``ratio`` = error / bar (inf for the exact checks)."""

    def __init__(self, msg, ratio=float("inf")):
        super(CheckFailed, self).__init__(msg)
        self.ratio = ratio


def check_output(e, split, x, w, w_exp, out, stats=None, seed=0):
    """Every check of one plan result: ``out`` the plan's whole NHWC output (its buffer NaN-filled before the run),
    ``stats`` its InstanceNorm sums, on any device.  -> (err/bar against the emulation, err/bar against fp32)."""
    from conv_emulation import EMU_BAR, FP32_BAR, STATS_BAR, stats_errors
    name = label(e, split)
    d = desc_of(e)
    _, cout, _ = real_dims(e)
    nan = torch.isnan(out)
    if bool(nan.any()):
        img, y, xx, c = (int(v) for v in nan.nonzero()[0])
        _, th, _, _, _, _, _ = schedule(d)
        f = 2 if d["transposed"] else 1
        raise CheckFailed("%s: %d output elements never written, the first at image %d (%d, %d) channel %d, tile (%d, %d)"
                             % (name, int(nan.sum()), img, y, xx, c, y // f // th, xx // f // TILE_W))
    if out.shape[-1] > cout:
        bad = out[..., cout:].contiguous().view(torch.int32) != 0
        if bool(bad.any()):
            raise CheckFailed("%s: output channels %d..%d are not +0 (%d elements)" % (name, cout, out.shape[-1],
                                                                                      int(bad.sum())))
    if stats is not None:
        e1, e2 = stats_errors(stats, out.permute(0, 3, 1, 2))
        if max(e1, e2) > STATS_BAR:
            raise CheckFailed("%s: statistics off their output's own sums by %.3e / %.3e (bar %.0e)"
                              % (name, e1, e2, STATS_BAR), max(e1, e2) / STATS_BAR)
    worst = [0.0, 0.0, 0.0, 0.0, None]                     # max |got - emu|, max |emu|, max |got - fp32|, max |fp32|, where
    for img, win in windows(e, seed):
        oy0, oy1, ox0, ox1 = win
        got = out[img, oy0:oy1, ox0:ox1, :cout].permute(2, 0, 1)[None].double().cpu()
        emu, f32 = reference(e, x, w, split, w_exp, img, win)
        diff = (got - emu).abs()
        if diff.max().item() > worst[0]:
            _, c, y, xx = np.unravel_index(int(diff.argmax()), diff.shape)
            worst[0], worst[4] = diff.max().item(), (img, oy0 + int(y), ox0 + int(xx), int(c))
        worst[1] = max(worst[1], emu.abs().max().item())
        worst[2] = max(worst[2], (got - f32.double()).abs().max().item())
        worst[3] = max(worst[3], f32.abs().max().item())
    emu_bar = EMU_BAR * max(1.0, (d["cin0"] + d["cin1"]) * d["kh"] * d["kw"] / EMU_K)
    emu_rel = worst[0] / (worst[1] + 1e-30) / emu_bar
    f32_rel = worst[2] / (worst[3] + 1e-30) / FP32_BAR[split]
    print("%s: err/bar %.3f vs emulation (worst at image, y, x, channel %s), %.3f vs fp32, %d windows"
          % (name, emu_rel, worst[4], f32_rel, len(windows(e, seed))))
    if emu_rel >= 1:
        raise CheckFailed("%s: %.3e of the output scale off the emulation at image, y, x, channel %s (bar %.1e)"
                          % (name, emu_rel * emu_bar, worst[4], emu_bar), emu_rel)
    if f32_rel >= 1:
        raise CheckFailed("%s: %.3e of the output scale off fp32 (bar %.0e)" % (name, f32_rel * FP32_BAR[split],
                                                                                FP32_BAR[split]), f32_rel)
    return emu_rel, f32_rel


# ------------------------------------------------------------------------------------------------------------- the census
# Regenerate with: print(format_census(entries_of(live_census()))) (test_conv_census_cpu.py prints the difference)
CENSUS = [
    # name, desc (DESC_FIELDS, split 0), weight shape, cout_pad, cin_pad, x, x1, stats, splits, (config, layer)
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 8 images = 2048 tiles, 15.5 per CTA
    Entry('rowk7x7_s1_8_64_n8_256x256', (8, 256, 256, 256, 256, 8, 0, 64, 7, 7, 1, 3, 1, 0, 0, 1, 264, 0, 0, -1),
          (64, 6, 7, 7), None, 8, (8, 262, 264, 8), None, True, (1,),
          (('unet_b8_256', 0),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 8 images = 1024 tiles, 7.8 per CTA
    Entry('conv3x3_s2_64_128_n8_128x128', (8, 256, 256, 128, 128, 64, 0, 128, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 64, 3, 3), None, None, (8, 256, 256, 64), None, True, (2, 1),
          (('unet_b8_256', 1),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 8 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s2_128_256_n8_64x64', (8, 128, 128, 64, 64, 128, 0, 256, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), None, None, (8, 128, 128, 128), None, True, (2, 1),
          (('unet_b8_256', 2),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 8 images = 256 tiles, 1.9 per CTA
    Entry('conv3x3_s2_256_512_n8_32x32', (8, 64, 64, 32, 32, 256, 0, 512, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (8, 64, 64, 256), None, True, (2, 1),
          (('unet_b8_256', 3),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 8 images = 256 tiles, 1.9 per CTA
    Entry('conv3x3_s1_512_512_n8_32x32', (8, 32, 32, 32, 32, 512, 0, 512, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (8, 32, 32, 512), None, True, (2, 1),
          (('unet_b8_256', 4), ('unet_b8_256', 5), ('unet_b8_256', 6), ('unet_b8_256', 7), ('unet_b8_256', 8), ('unet_b8_256', 9), ('unet_b8_256', 10), ('unet_b8_256', 11), ('unet_b8_256', 12), ('unet_b8_256', 13), ('unet_b8_256', 14), ('unet_b8_256', 15),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 2 N tiles x 8 images = 128 tiles, 1.0 per CTA
    Entry('convT3x3_s2_512_256_n8_64x64', (8, 32, 32, 64, 64, 512, 0, 256, 3, 3, 2, 1, 1, 1, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (8, 32, 32, 512), None, True, (2, 1),
          (('unet_b8_256', 16),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 8 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s1_256+256_256_n8_64x64', (8, 64, 64, 64, 64, 256, 256, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 512, 3, 3), None, None, (8, 64, 64, 256), (8, 64, 64, 256), True, (2, 1),
          (('unet_b8_256', 17),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 4 N tiles x 8 images = 1024 tiles, 7.8 per CTA
    Entry('convTm3x3_s2_256_128_n8_128x128', (8, 64, 64, 128, 128, 256, 0, 128, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (512, 256, 2, 2), None, None, (8, 64, 64, 256), None, True, (2, 1),
          (('unet_b8_256', 18),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 8 images = 1024 tiles, 7.8 per CTA
    Entry('conv3x3_s1_128+128_128_n8_128x128', (8, 128, 128, 128, 128, 128, 128, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 256, 3, 3), None, None, (8, 128, 128, 128), (8, 128, 128, 128), True, (2, 1),
          (('unet_b8_256', 19),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 2 N tiles x 8 images = 2048 tiles, 15.5 per CTA
    Entry('convTm3x3_s2_128_64_n8_256x256', (8, 128, 128, 256, 256, 128, 0, 64, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (256, 128, 2, 2), None, None, (8, 128, 128, 128), None, True, (2, 1),
          (('unet_b8_256', 20),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 8 images = 2048 tiles, 15.5 per CTA
    Entry('conv3x3_s1_64+64_64_n8_256x256', (8, 256, 256, 256, 256, 64, 64, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 128, 3, 3), None, None, (8, 256, 256, 64), (8, 256, 256, 64), True, (2, 1),
          (('unet_b8_256', 21),)),
    # N tile 32, 16x8 tiles, 16 x 32 x 1 N tiles x 8 images = 4096 tiles, 31.0 per CTA
    Entry('conv7x1_s1_64_32_n8_256x256_pw0_nt32', (8, 256, 256, 256, 256, 64, 0, 32, 7, 1, 1, 3, 1, 0, 0, 0, 0, 32, 0, 0),
          (32, 64, 7, 1), None, None, (8, 256, 256, 64), None, False, (2, 1),
          (('unet_b8_256', 22),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 16 images = 4096 tiles, 31.0 per CTA
    Entry('rowk7x7_s1_8_64_n16_256x256', (16, 256, 256, 256, 256, 8, 0, 64, 7, 7, 1, 3, 1, 0, 0, 1, 264, 0, 0, -1),
          (64, 6, 7, 7), None, 8, (16, 262, 264, 8), None, True, (1,),
          (('unet_b16_256', 0),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 16 images = 2048 tiles, 15.5 per CTA
    Entry('conv3x3_s2_64_128_n16_128x128', (16, 256, 256, 128, 128, 64, 0, 128, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 64, 3, 3), None, None, (16, 256, 256, 64), None, True, (2, 1),
          (('unet_b16_256', 1),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 16 images = 1024 tiles, 7.8 per CTA
    Entry('conv3x3_s2_128_256_n16_64x64', (16, 128, 128, 64, 64, 128, 0, 256, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), None, None, (16, 128, 128, 128), None, True, (2, 1),
          (('unet_b16_256', 2),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 16 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s2_256_512_n16_32x32', (16, 64, 64, 32, 32, 256, 0, 512, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (16, 64, 64, 256), None, True, (2, 1),
          (('unet_b16_256', 3),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 16 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s1_512_512_n16_32x32', (16, 32, 32, 32, 32, 512, 0, 512, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (16, 32, 32, 512), None, True, (2, 1),
          (('unet_b16_256', 4), ('unet_b16_256', 5), ('unet_b16_256', 6), ('unet_b16_256', 7), ('unet_b16_256', 8), ('unet_b16_256', 9), ('unet_b16_256', 10), ('unet_b16_256', 11), ('unet_b16_256', 12), ('unet_b16_256', 13), ('unet_b16_256', 14), ('unet_b16_256', 15),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 2 N tiles x 16 images = 256 tiles, 1.9 per CTA
    Entry('convT3x3_s2_512_256_n16_64x64', (16, 32, 32, 64, 64, 512, 0, 256, 3, 3, 2, 1, 1, 1, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (16, 32, 32, 512), None, True, (2, 1),
          (('unet_b16_256', 16),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 16 images = 1024 tiles, 7.8 per CTA
    Entry('conv3x3_s1_256+256_256_n16_64x64', (16, 64, 64, 64, 64, 256, 256, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 512, 3, 3), None, None, (16, 64, 64, 256), (16, 64, 64, 256), True, (2, 1),
          (('unet_b16_256', 17),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 4 N tiles x 16 images = 2048 tiles, 15.5 per CTA
    Entry('convTm3x3_s2_256_128_n16_128x128', (16, 64, 64, 128, 128, 256, 0, 128, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (512, 256, 2, 2), None, None, (16, 64, 64, 256), None, True, (2, 1),
          (('unet_b16_256', 18),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 16 images = 2048 tiles, 15.5 per CTA
    Entry('conv3x3_s1_128+128_128_n16_128x128', (16, 128, 128, 128, 128, 128, 128, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 256, 3, 3), None, None, (16, 128, 128, 128), (16, 128, 128, 128), True, (2, 1),
          (('unet_b16_256', 19),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 2 N tiles x 16 images = 4096 tiles, 31.0 per CTA
    Entry('convTm3x3_s2_128_64_n16_256x256', (16, 128, 128, 256, 256, 128, 0, 64, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (256, 128, 2, 2), None, None, (16, 128, 128, 128), None, True, (2, 1),
          (('unet_b16_256', 20),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 16 images = 4096 tiles, 31.0 per CTA
    Entry('conv3x3_s1_64+64_64_n16_256x256', (16, 256, 256, 256, 256, 64, 64, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 128, 3, 3), None, None, (16, 256, 256, 64), (16, 256, 256, 64), True, (2, 1),
          (('unet_b16_256', 21),)),
    # N tile 32, 16x8 tiles, 16 x 32 x 1 N tiles x 16 images = 8192 tiles, 62.1 per CTA
    Entry('conv7x1_s1_64_32_n16_256x256_pw0_nt32', (16, 256, 256, 256, 256, 64, 0, 32, 7, 1, 1, 3, 1, 0, 0, 0, 0, 32, 0, 0),
          (32, 64, 7, 1), None, None, (16, 256, 256, 64), None, False, (2, 1),
          (('unet_b16_256', 22),)),
    # N tile 64, 32x8 tiles, 16 x 64 x 1 N tiles x 4 images = 4096 tiles, 31.0 per CTA
    Entry('rowk7x7_s1_8_64_n4_512x512', (4, 512, 512, 512, 512, 8, 0, 64, 7, 7, 1, 3, 1, 0, 0, 1, 520, 0, 0, -1),
          (64, 6, 7, 7), None, 8, (4, 518, 520, 8), None, True, (1,),
          (('unet_b4_512', 0),)),
    # N tile 128, 16x8 tiles, 16 x 32 x 1 N tiles x 4 images = 2048 tiles, 15.5 per CTA
    Entry('conv3x3_s2_64_128_n4_256x256', (4, 512, 512, 256, 256, 64, 0, 128, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 64, 3, 3), None, None, (4, 512, 512, 64), None, True, (2, 1),
          (('unet_b4_512', 1),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 2 N tiles x 4 images = 1024 tiles, 7.8 per CTA
    Entry('conv3x3_s2_128_256_n4_128x128', (4, 256, 256, 128, 128, 128, 0, 256, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), None, None, (4, 256, 256, 128), None, True, (2, 1),
          (('unet_b4_512', 2),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 4 N tiles x 4 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s2_256_512_n4_64x64', (4, 128, 128, 64, 64, 256, 0, 512, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (4, 128, 128, 256), None, True, (2, 1),
          (('unet_b4_512', 3),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 4 N tiles x 4 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s1_512_512_n4_64x64', (4, 64, 64, 64, 64, 512, 0, 512, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (4, 64, 64, 512), None, True, (2, 1),
          (('unet_b4_512', 4), ('unet_b4_512', 5), ('unet_b4_512', 6), ('unet_b4_512', 7), ('unet_b4_512', 8), ('unet_b4_512', 9), ('unet_b4_512', 10), ('unet_b4_512', 11), ('unet_b4_512', 12), ('unet_b4_512', 13), ('unet_b4_512', 14), ('unet_b4_512', 15),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 4 images = 256 tiles, 1.9 per CTA
    Entry('convT3x3_s2_512_256_n4_128x128', (4, 64, 64, 128, 128, 512, 0, 256, 3, 3, 2, 1, 1, 1, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (4, 64, 64, 512), None, True, (2, 1),
          (('unet_b4_512', 16),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 2 N tiles x 4 images = 1024 tiles, 7.8 per CTA
    Entry('conv3x3_s1_256+256_256_n4_128x128', (4, 128, 128, 128, 128, 256, 256, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 512, 3, 3), None, None, (4, 128, 128, 256), (4, 128, 128, 256), True, (2, 1),
          (('unet_b4_512', 17),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 4 N tiles x 4 images = 2048 tiles, 15.5 per CTA
    Entry('convTm3x3_s2_256_128_n4_256x256', (4, 128, 128, 256, 256, 256, 0, 128, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (512, 256, 2, 2), None, None, (4, 128, 128, 256), None, True, (2, 1),
          (('unet_b4_512', 18),)),
    # N tile 128, 16x8 tiles, 16 x 32 x 1 N tiles x 4 images = 2048 tiles, 15.5 per CTA
    Entry('conv3x3_s1_128+128_128_n4_256x256', (4, 256, 256, 256, 256, 128, 128, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 256, 3, 3), None, None, (4, 256, 256, 128), (4, 256, 256, 128), True, (2, 1),
          (('unet_b4_512', 19),)),
    # N tile 128, 16x8 tiles, 16 x 32 x 2 N tiles x 4 images = 4096 tiles, 31.0 per CTA
    Entry('convTm3x3_s2_128_64_n4_512x512', (4, 256, 256, 512, 512, 128, 0, 64, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (256, 128, 2, 2), None, None, (4, 256, 256, 128), None, True, (2, 1),
          (('unet_b4_512', 20),)),
    # N tile 64, 32x8 tiles, 16 x 64 x 1 N tiles x 4 images = 4096 tiles, 31.0 per CTA
    Entry('conv3x3_s1_64+64_64_n4_512x512', (4, 512, 512, 512, 512, 64, 64, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 128, 3, 3), None, None, (4, 512, 512, 64), (4, 512, 512, 64), True, (2, 1),
          (('unet_b4_512', 21),)),
    # N tile 32, 16x8 tiles, 32 x 64 x 1 N tiles x 4 images = 8192 tiles, 62.1 per CTA
    Entry('conv7x1_s1_64_32_n4_512x512_pw0_nt32', (4, 512, 512, 512, 512, 64, 0, 32, 7, 1, 1, 3, 1, 0, 0, 0, 0, 32, 0, 0),
          (32, 64, 7, 1), None, None, (4, 512, 512, 64), None, False, (2, 1),
          (('unet_b4_512', 22),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 1 images = 256 tiles, 1.9 per CTA
    Entry('rowk7x7_s1_8_64_n1_256x256_v1', (1, 256, 256, 256, 256, 8, 0, 64, 7, 7, 1, 3, 1, 0, 0, 1, 264, 0, 0, -1),
          (64, 6, 7, 7), None, 8, (1, 262, 264, 8), None, True, (1,),
          (('src_b1_256', 0),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv3x3_s2_64_128_n1_128x128', (1, 256, 256, 128, 128, 64, 0, 128, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 64, 3, 3), None, None, (1, 256, 256, 64), None, True, (2, 1),
          (('src_b1_256', 1), ('bg_b1_256', 1),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s2_128_256_n1_64x64', (1, 128, 128, 64, 64, 128, 0, 256, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), None, None, (1, 128, 128, 128), None, True, (2, 1),
          (('src_b1_256', 2), ('bg_b1_256', 2),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv3x3_s2_256_512_n1_32x32', (1, 64, 64, 32, 32, 256, 0, 512, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (1, 64, 64, 256), None, True, (2, 1),
          (('src_b1_256', 3), ('bg_b1_256', 3),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv3x3_s1_512_512_n1_32x32', (1, 32, 32, 32, 32, 512, 0, 512, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (1, 32, 32, 512), None, True, (2, 1),
          (('src_b1_256', 4), ('src_b1_256', 5), ('src_b1_256', 6), ('src_b1_256', 7), ('src_b1_256', 8), ('src_b1_256', 9), ('src_b1_256', 10), ('src_b1_256', 11), ('src_b1_256', 12), ('src_b1_256', 13), ('src_b1_256', 14), ('src_b1_256', 15), ('bg_b1_256', 4), ('bg_b1_256', 5), ('bg_b1_256', 6), ('bg_b1_256', 7), ('bg_b1_256', 8), ('bg_b1_256', 9), ('bg_b1_256', 10), ('bg_b1_256', 11), ('bg_b1_256', 12), ('bg_b1_256', 13), ('bg_b1_256', 14), ('bg_b1_256', 15),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 2 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('convT3x3_s2_512_256_n1_64x64', (1, 32, 32, 64, 64, 512, 0, 256, 3, 3, 2, 1, 1, 1, 0, 0, 0, 0, 0, -1),
          (512, 256, 3, 3), None, None, (1, 32, 32, 512), None, True, (2, 1),
          (('src_b1_256', 16), ('bg_b1_256', 16),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_256+256_256_n1_64x64', (1, 64, 64, 64, 64, 256, 256, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 512, 3, 3), None, None, (1, 64, 64, 256), (1, 64, 64, 256), True, (2, 1),
          (('src_b1_256', 17),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 4 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('convTm3x3_s2_256_128_n1_128x128', (1, 64, 64, 128, 128, 256, 0, 128, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (512, 256, 2, 2), None, None, (1, 64, 64, 256), None, True, (2, 1),
          (('src_b1_256', 18), ('bg_b1_256', 17),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128+128_128_n1_128x128', (1, 128, 128, 128, 128, 128, 128, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 256, 3, 3), None, None, (1, 128, 128, 128), (1, 128, 128, 128), True, (2, 1),
          (('src_b1_256', 19),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 2 N tiles x 1 images = 256 tiles, 1.9 per CTA
    Entry('convTm3x3_s2_128_64_n1_256x256', (1, 128, 128, 256, 256, 128, 0, 64, 3, 3, 2, 1, 1, 2, 0, 0, 0, 0, 0, -1),
          (256, 128, 2, 2), None, None, (1, 128, 128, 128), None, True, (2, 1),
          (('src_b1_256', 20), ('bg_b1_256', 18),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 1 images = 256 tiles, 1.9 per CTA
    Entry('conv3x3_s1_64+64_64_n1_256x256', (1, 256, 256, 256, 256, 64, 64, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 128, 3, 3), None, None, (1, 256, 256, 64), (1, 256, 256, 64), True, (2, 1),
          (('src_b1_256', 21),)),
    # N tile 32, 16x8 tiles, 16 x 32 x 1 N tiles x 1 images = 512 tiles, 3.9 per CTA
    Entry('conv7x1_s1_64_32_n1_256x256_pw0_nt32', (1, 256, 256, 256, 256, 64, 0, 32, 7, 1, 1, 3, 1, 0, 0, 0, 0, 32, 0, 0),
          (32, 64, 7, 1), None, None, (1, 256, 256, 64), None, False, (2, 1),
          (('src_b1_256', 22), ('bg_b1_256', 19),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 1 images = 256 tiles, 1.9 per CTA
    Entry('rowk7x7_s1_8_64_n1_256x256_v2', (1, 256, 256, 256, 256, 8, 0, 64, 7, 7, 1, 3, 1, 0, 0, 1, 264, 0, 0, -1),
          (64, 4, 7, 7), None, 8, (1, 262, 264, 8), None, True, (1,),
          (('bg_b1_256', 0),)),
    # N tile 64, 32x8 tiles, 2 x 7 x 1 N tiles x 1 images = 14 tiles, 1.0 per CTA
    Entry('conv1x1_s1_64_64_n1_56x56', (1, 56, 56, 56, 56, 64, 0, 64, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 1, 1), None, None, (1, 56, 56, 64), None, False, (2, 1),
          (('hmr_b1', 0),)),
    # N tile 64, 32x8 tiles, 2 x 7 x 1 N tiles x 1 images = 14 tiles, 1.0 per CTA
    Entry('conv3x3_s1_64_64_n1_56x56', (1, 56, 56, 56, 56, 64, 0, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 3, 3), None, None, (1, 56, 56, 64), None, False, (2, 1),
          (('hmr_b1', 1), ('hmr_b1', 5),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 2 N tiles x 1 images = 56 tiles, 1.0 per CTA
    Entry('conv1x1_s1_64_256_n1_56x56', (1, 56, 56, 56, 56, 64, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 64, 1, 1), None, None, (1, 56, 56, 64), None, False, (2, 1),
          (('hmr_b1', 2), ('hmr_b1', 3), ('hmr_b1', 6),)),
    # N tile 64, 32x8 tiles, 2 x 7 x 1 N tiles x 1 images = 14 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_64_n1_56x56', (1, 56, 56, 56, 56, 256, 0, 64, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 256, 1, 1), None, None, (1, 56, 56, 256), None, False, (2, 1),
          (('hmr_b1', 4), ('hmr_b1', 7),)),
    # N tile 64, 32x8 tiles, 1 x 4 x 1 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv3x3_s2_64_64_n1_28x28', (1, 56, 56, 28, 28, 64, 0, 64, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 3, 3), None, None, (1, 56, 56, 64), None, False, (2, 1),
          (('hmr_b1', 8),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 2 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('conv1x1_s1_64_256_n1_28x28', (1, 28, 28, 28, 28, 64, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 64, 1, 1), None, None, (1, 28, 28, 64), None, False, (2, 1),
          (('hmr_b1', 9),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 1 N tiles x 1 images = 8 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_128_n1_28x28', (1, 28, 28, 28, 28, 256, 0, 128, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 256, 1, 1), None, None, (1, 28, 28, 256), None, False, (2, 1),
          (('hmr_b1', 10),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 1 N tiles x 1 images = 8 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_128_n1_28x28', (1, 28, 28, 28, 28, 128, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 128, 3, 3), None, None, (1, 28, 28, 128), None, False, (2, 1),
          (('hmr_b1', 11), ('hmr_b1', 15), ('hmr_b1', 18),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv1x1_s1_128_512_n1_28x28', (1, 28, 28, 28, 28, 128, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 128, 1, 1), None, None, (1, 28, 28, 128), None, False, (2, 1),
          (('hmr_b1', 12), ('hmr_b1', 16), ('hmr_b1', 19),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_512_n1_28x28', (1, 28, 28, 28, 28, 256, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 256, 1, 1), None, None, (1, 28, 28, 256), None, False, (2, 1),
          (('hmr_b1', 13),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 1 N tiles x 1 images = 8 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_128_n1_28x28', (1, 28, 28, 28, 28, 512, 0, 128, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 512, 1, 1), None, None, (1, 28, 28, 512), None, False, (2, 1),
          (('hmr_b1', 14), ('hmr_b1', 17), ('hmr_b1', 20),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 1 N tiles x 1 images = 2 tiles, 1.0 per CTA
    Entry('conv3x3_s2_128_128_n1_14x14', (1, 28, 28, 14, 14, 128, 0, 128, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 128, 3, 3), None, None, (1, 28, 28, 128), None, False, (2, 1),
          (('hmr_b1', 21),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 4 N tiles x 1 images = 8 tiles, 1.0 per CTA
    Entry('conv1x1_s1_128_512_n1_14x14', (1, 14, 14, 14, 14, 128, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 128, 1, 1), None, None, (1, 14, 14, 128), None, False, (2, 1),
          (('hmr_b1', 22),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_256_n1_14x14', (1, 14, 14, 14, 14, 512, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 512, 1, 1), None, None, (1, 14, 14, 512), None, False, (2, 1),
          (('hmr_b1', 23),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv3x3_s1_256_256_n1_14x14', (1, 14, 14, 14, 14, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 14, 14, 256), None, False, (2, 1),
          (('hmr_b1', 24), ('hmr_b1', 28), ('hmr_b1', 31), ('hmr_b1', 34), ('hmr_b1', 37),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 8 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_1024_n1_14x14', (1, 14, 14, 14, 14, 256, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 256, 1, 1), None, None, (1, 14, 14, 256), None, False, (2, 1),
          (('hmr_b1', 25), ('hmr_b1', 29), ('hmr_b1', 32), ('hmr_b1', 35), ('hmr_b1', 38),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 8 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_1024_n1_14x14', (1, 14, 14, 14, 14, 512, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 512, 1, 1), None, None, (1, 14, 14, 512), None, False, (2, 1),
          (('hmr_b1', 26),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_256_n1_14x14', (1, 14, 14, 14, 14, 1024, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 1024, 1, 1), None, None, (1, 14, 14, 1024), None, False, (2, 1),
          (('hmr_b1', 27), ('hmr_b1', 30), ('hmr_b1', 33), ('hmr_b1', 36), ('hmr_b1', 39),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 2 N tiles x 1 images = 2 tiles, 1.0 per CTA
    Entry('conv3x3_s2_256_256_n1_7x7', (1, 14, 14, 7, 7, 256, 0, 256, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 14, 14, 256), None, False, (2, 1),
          (('hmr_b1', 40),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 8 N tiles x 1 images = 8 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_1024_n1_7x7', (1, 7, 7, 7, 7, 256, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 256, 1, 1), None, None, (1, 7, 7, 256), None, False, (2, 1),
          (('hmr_b1', 41),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 4 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_512_n1_7x7', (1, 7, 7, 7, 7, 1024, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 1024, 1, 1), None, None, (1, 7, 7, 1024), None, False, (2, 1),
          (('hmr_b1', 42),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 4 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv3x3_s1_512_512_n1_7x7', (1, 7, 7, 7, 7, 512, 0, 512, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (1, 7, 7, 512), None, False, (2, 1),
          (('hmr_b1', 43), ('hmr_b1', 47), ('hmr_b1', 50),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 16 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_2048_n1_7x7', (1, 7, 7, 7, 7, 512, 0, 2048, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (2048, 512, 1, 1), None, None, (1, 7, 7, 512), None, False, (2, 1),
          (('hmr_b1', 44), ('hmr_b1', 48), ('hmr_b1', 51),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 16 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_2048_n1_7x7', (1, 7, 7, 7, 7, 1024, 0, 2048, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (2048, 1024, 1, 1), None, None, (1, 7, 7, 1024), None, False, (2, 1),
          (('hmr_b1', 45),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 4 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv1x1_s1_2048_512_n1_7x7', (1, 7, 7, 7, 7, 2048, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 2048, 1, 1), None, None, (1, 7, 7, 2048), None, False, (2, 1),
          (('hmr_b1', 46), ('hmr_b1', 49),)),
    # N tile 64, 32x8 tiles, 2 x 7 x 1 N tiles x 16 images = 224 tiles, 1.7 per CTA
    Entry('conv1x1_s1_64_64_n16_56x56', (16, 56, 56, 56, 56, 64, 0, 64, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 1, 1), None, None, (16, 56, 56, 64), None, False, (2, 1),
          (('hmr_b16', 0),)),
    # N tile 64, 32x8 tiles, 2 x 7 x 1 N tiles x 16 images = 224 tiles, 1.7 per CTA
    Entry('conv3x3_s1_64_64_n16_56x56', (16, 56, 56, 56, 56, 64, 0, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 3, 3), None, None, (16, 56, 56, 64), None, False, (2, 1),
          (('hmr_b16', 1), ('hmr_b16', 5),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 2 N tiles x 16 images = 896 tiles, 6.8 per CTA
    Entry('conv1x1_s1_64_256_n16_56x56', (16, 56, 56, 56, 56, 64, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 64, 1, 1), None, None, (16, 56, 56, 64), None, False, (2, 1),
          (('hmr_b16', 2), ('hmr_b16', 3), ('hmr_b16', 6),)),
    # N tile 64, 32x8 tiles, 2 x 7 x 1 N tiles x 16 images = 224 tiles, 1.7 per CTA
    Entry('conv1x1_s1_256_64_n16_56x56', (16, 56, 56, 56, 56, 256, 0, 64, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 256, 1, 1), None, None, (16, 56, 56, 256), None, False, (2, 1),
          (('hmr_b16', 4), ('hmr_b16', 7),)),
    # N tile 64, 32x8 tiles, 1 x 4 x 1 N tiles x 16 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s2_64_64_n16_28x28', (16, 56, 56, 28, 28, 64, 0, 64, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 3, 3), None, None, (16, 56, 56, 64), None, False, (2, 1),
          (('hmr_b16', 8),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 2 N tiles x 16 images = 256 tiles, 1.9 per CTA
    Entry('conv1x1_s1_64_256_n16_28x28', (16, 28, 28, 28, 28, 64, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 64, 1, 1), None, None, (16, 28, 28, 64), None, False, (2, 1),
          (('hmr_b16', 9),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 1 N tiles x 16 images = 128 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_128_n16_28x28', (16, 28, 28, 28, 28, 256, 0, 128, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 256, 1, 1), None, None, (16, 28, 28, 256), None, False, (2, 1),
          (('hmr_b16', 10),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 1 N tiles x 16 images = 128 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_128_n16_28x28', (16, 28, 28, 28, 28, 128, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 128, 3, 3), None, None, (16, 28, 28, 128), None, False, (2, 1),
          (('hmr_b16', 11), ('hmr_b16', 15), ('hmr_b16', 18),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 16 images = 512 tiles, 3.9 per CTA
    Entry('conv1x1_s1_128_512_n16_28x28', (16, 28, 28, 28, 28, 128, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 128, 1, 1), None, None, (16, 28, 28, 128), None, False, (2, 1),
          (('hmr_b16', 12), ('hmr_b16', 16), ('hmr_b16', 19),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 16 images = 512 tiles, 3.9 per CTA
    Entry('conv1x1_s1_256_512_n16_28x28', (16, 28, 28, 28, 28, 256, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 256, 1, 1), None, None, (16, 28, 28, 256), None, False, (2, 1),
          (('hmr_b16', 13),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 1 N tiles x 16 images = 128 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_128_n16_28x28', (16, 28, 28, 28, 28, 512, 0, 128, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 512, 1, 1), None, None, (16, 28, 28, 512), None, False, (2, 1),
          (('hmr_b16', 14), ('hmr_b16', 17), ('hmr_b16', 20),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 1 N tiles x 16 images = 32 tiles, 1.0 per CTA
    Entry('conv3x3_s2_128_128_n16_14x14', (16, 28, 28, 14, 14, 128, 0, 128, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 128, 3, 3), None, None, (16, 28, 28, 128), None, False, (2, 1),
          (('hmr_b16', 21),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 4 N tiles x 16 images = 128 tiles, 1.0 per CTA
    Entry('conv1x1_s1_128_512_n16_14x14', (16, 14, 14, 14, 14, 128, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 128, 1, 1), None, None, (16, 14, 14, 128), None, False, (2, 1),
          (('hmr_b16', 22),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 16 images = 64 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_256_n16_14x14', (16, 14, 14, 14, 14, 512, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 512, 1, 1), None, None, (16, 14, 14, 512), None, False, (2, 1),
          (('hmr_b16', 23),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 16 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_256_256_n16_14x14', (16, 14, 14, 14, 14, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (16, 14, 14, 256), None, False, (2, 1),
          (('hmr_b16', 24), ('hmr_b16', 28), ('hmr_b16', 31), ('hmr_b16', 34), ('hmr_b16', 37),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 8 N tiles x 16 images = 256 tiles, 1.9 per CTA
    Entry('conv1x1_s1_256_1024_n16_14x14', (16, 14, 14, 14, 14, 256, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 256, 1, 1), None, None, (16, 14, 14, 256), None, False, (2, 1),
          (('hmr_b16', 25), ('hmr_b16', 29), ('hmr_b16', 32), ('hmr_b16', 35), ('hmr_b16', 38),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 8 N tiles x 16 images = 256 tiles, 1.9 per CTA
    Entry('conv1x1_s1_512_1024_n16_14x14', (16, 14, 14, 14, 14, 512, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 512, 1, 1), None, None, (16, 14, 14, 512), None, False, (2, 1),
          (('hmr_b16', 26),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 16 images = 64 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_256_n16_14x14', (16, 14, 14, 14, 14, 1024, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 1024, 1, 1), None, None, (16, 14, 14, 1024), None, False, (2, 1),
          (('hmr_b16', 27), ('hmr_b16', 30), ('hmr_b16', 33), ('hmr_b16', 36), ('hmr_b16', 39),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 2 N tiles x 16 images = 32 tiles, 1.0 per CTA
    Entry('conv3x3_s2_256_256_n16_7x7', (16, 14, 14, 7, 7, 256, 0, 256, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (16, 14, 14, 256), None, False, (2, 1),
          (('hmr_b16', 40),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 8 N tiles x 16 images = 128 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_1024_n16_7x7', (16, 7, 7, 7, 7, 256, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 256, 1, 1), None, None, (16, 7, 7, 256), None, False, (2, 1),
          (('hmr_b16', 41),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 4 N tiles x 16 images = 64 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_512_n16_7x7', (16, 7, 7, 7, 7, 1024, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 1024, 1, 1), None, None, (16, 7, 7, 1024), None, False, (2, 1),
          (('hmr_b16', 42),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 4 N tiles x 16 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_512_512_n16_7x7', (16, 7, 7, 7, 7, 512, 0, 512, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (16, 7, 7, 512), None, False, (2, 1),
          (('hmr_b16', 43), ('hmr_b16', 47), ('hmr_b16', 50),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 16 N tiles x 16 images = 256 tiles, 1.9 per CTA
    Entry('conv1x1_s1_512_2048_n16_7x7', (16, 7, 7, 7, 7, 512, 0, 2048, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (2048, 512, 1, 1), None, None, (16, 7, 7, 512), None, False, (2, 1),
          (('hmr_b16', 44), ('hmr_b16', 48), ('hmr_b16', 51),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 16 N tiles x 16 images = 256 tiles, 1.9 per CTA
    Entry('conv1x1_s1_1024_2048_n16_7x7', (16, 7, 7, 7, 7, 1024, 0, 2048, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (2048, 1024, 1, 1), None, None, (16, 7, 7, 1024), None, False, (2, 1),
          (('hmr_b16', 45),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 4 N tiles x 16 images = 64 tiles, 1.0 per CTA
    Entry('conv1x1_s1_2048_512_n16_7x7', (16, 7, 7, 7, 7, 2048, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 2048, 1, 1), None, None, (16, 7, 7, 2048), None, False, (2, 1),
          (('hmr_b16', 46), ('hmr_b16', 49),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 1 images = 256 tiles, 1.9 per CTA
    Entry('conv5x5_s1_64_64_n1_256x256', (1, 256, 256, 256, 256, 64, 0, 64, 5, 5, 1, 2, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 4, 5, 5), 64, 64, (1, 256, 256, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 0), ('inpaintor_b1_256', 17),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv4x4_s2_64_128_n1_128x128_p1', (1, 256, 256, 128, 128, 64, 0, 128, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 32, 4, 4), 128, 64, (1, 256, 256, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 1),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv3x3_s1_64_128_n1_128x128_v1', (1, 128, 128, 128, 128, 64, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 64, 3, 3), 128, 64, (1, 128, 128, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 2), ('inpaintor_b1_256', 13), ('inpaintor_b1_256', 32),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv4x4_s2_64_256_n1_64x64_p1', (1, 128, 128, 64, 64, 64, 0, 256, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 64, 4, 4), 256, 64, (1, 128, 128, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 3),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_256_n1_64x64', (1, 64, 64, 64, 64, 128, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), 256, 128, (1, 64, 64, 128), None, False, (2, 1),
          (('inpaintor_b1_256', 4), ('inpaintor_b1_256', 5), ('inpaintor_b1_256', 10), ('inpaintor_b1_256', 11), ('inpaintor_b1_256', 22), ('inpaintor_b1_256', 23), ('inpaintor_b1_256', 29), ('inpaintor_b1_256', 30),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_256_n1_64x64_p2_d2', (1, 64, 64, 64, 64, 128, 0, 256, 3, 3, 1, 2, 2, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), 256, 128, (1, 64, 64, 128), None, False, (2, 1),
          (('inpaintor_b1_256', 6), ('inpaintor_b1_256', 24),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_256_n1_64x64_p4_d4', (1, 64, 64, 64, 64, 128, 0, 256, 3, 3, 1, 4, 4, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), 256, 128, (1, 64, 64, 128), None, False, (2, 1),
          (('inpaintor_b1_256', 7), ('inpaintor_b1_256', 25),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_256_n1_64x64_p8_d8', (1, 64, 64, 64, 64, 128, 0, 256, 3, 3, 1, 8, 8, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), 256, 128, (1, 64, 64, 128), None, False, (2, 1),
          (('inpaintor_b1_256', 8), ('inpaintor_b1_256', 26),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_256_n1_64x64_p16_d16', (1, 64, 64, 64, 64, 128, 0, 256, 3, 3, 1, 16, 16, 0, 0, 0, 0, 0, 0, -1),
          (256, 128, 3, 3), 256, 128, (1, 64, 64, 128), None, False, (2, 1),
          (('inpaintor_b1_256', 9), ('inpaintor_b1_256', 27),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_128_n1_128x128', (1, 128, 128, 128, 128, 128, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 128, 3, 3), 128, 128, (1, 128, 128, 128), None, False, (2, 1),
          (('inpaintor_b1_256', 12), ('inpaintor_b1_256', 31),)),
    # N tile 64, 32x8 tiles, 8 x 32 x 1 N tiles x 1 images = 256 tiles, 1.9 per CTA
    Entry('conv3x3_s1_64_64_n1_256x256', (1, 256, 256, 256, 256, 64, 0, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 3, 3), 64, 64, (1, 256, 256, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 14), ('inpaintor_b1_256', 33),)),
    # N tile 32, 16x8 tiles, 16 x 32 x 1 N tiles x 1 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s1_64_32_n1_256x256', (1, 256, 256, 256, 256, 64, 0, 32, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (32, 32, 3, 3), 32, 64, (1, 256, 256, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 15), ('inpaintor_b1_256', 34),)),
    # N tile 16, 16x8 tiles, 16 x 32 x 1 N tiles x 1 images = 512 tiles, 3.9 per CTA
    Entry('conv3x3_s1_64_16_n1_256x256', (1, 256, 256, 256, 256, 64, 0, 16, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (6, 16, 3, 3), 16, 64, (1, 256, 256, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 16), ('inpaintor_b1_256', 35),)),
    # N tile 64, 32x8 tiles, 4 x 16 x 1 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv4x4_s2_64_64_n1_128x128_p1', (1, 256, 256, 128, 128, 64, 0, 64, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 32, 4, 4), 64, 64, (1, 256, 256, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 18),)),
    # N tile 128, 16x8 tiles, 8 x 16 x 1 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv3x3_s1_64_128_n1_128x128_v2', (1, 128, 128, 128, 128, 64, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 32, 3, 3), 128, 64, (1, 128, 128, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 19),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 1 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv4x4_s2_64_128_n1_64x64_p1', (1, 128, 128, 64, 64, 64, 0, 128, 4, 4, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 64, 4, 4), 128, 64, (1, 128, 128, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 20),)),
    # N tile 128, 16x8 tiles, 4 x 8 x 2 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv3x3_s1_64_256_n1_64x64', (1, 64, 64, 64, 64, 64, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 64, 3, 3), 256, 64, (1, 64, 64, 64), None, False, (2, 1),
          (('inpaintor_b1_256', 21),)),
    # N tile 32, 16x8 tiles, 4 x 8 x 5 N tiles x 1 images = 160 tiles, 1.2 per CTA
    Entry('conv1x1_s1_128_160_n1_64x64', (1, 64, 64, 64, 64, 128, 0, 160, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (160, 128, 1, 1), 160, 128, (1, 64, 64, 128), None, False, (2, 1),
          (('inpaintor_b1_256', 28),)),
    # N tile 64, 32x8 tiles, 7 x 25 x 1 N tiles x 1 images = 175 tiles, 1.3 per CTA
    Entry('conv1x1_s1_64_64_n1_200x200', (1, 200, 200, 200, 200, 64, 0, 64, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 1, 1), None, None, (1, 200, 200, 64), None, False, (1,),
          (('detector_256', 0), ('detector_512', 0),)),
    # N tile 64, 32x8 tiles, 7 x 25 x 1 N tiles x 1 images = 175 tiles, 1.3 per CTA
    Entry('conv3x3_s1_64_64_n1_200x200', (1, 200, 200, 200, 200, 64, 0, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 64, 3, 3), None, None, (1, 200, 200, 64), None, False, (1,),
          (('detector_256', 1), ('detector_256', 5), ('detector_256', 8), ('detector_512', 1), ('detector_512', 5), ('detector_512', 8),)),
    # N tile 128, 16x8 tiles, 13 x 25 x 2 N tiles x 1 images = 650 tiles, 4.9 per CTA
    Entry('conv1x1_s1_64_256_n1_200x200', (1, 200, 200, 200, 200, 64, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 64, 1, 1), None, None, (1, 200, 200, 64), None, False, (1,),
          (('detector_256', 2), ('detector_256', 3), ('detector_256', 6), ('detector_256', 9), ('detector_512', 2), ('detector_512', 3), ('detector_512', 6), ('detector_512', 9),)),
    # N tile 64, 32x8 tiles, 7 x 25 x 1 N tiles x 1 images = 175 tiles, 1.3 per CTA
    Entry('conv1x1_s1_256_64_n1_200x200', (1, 200, 200, 200, 200, 256, 0, 64, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (64, 256, 1, 1), None, None, (1, 200, 200, 256), None, False, (1,),
          (('detector_256', 4), ('detector_256', 7), ('detector_512', 4), ('detector_512', 7),)),
    # N tile 128, 16x8 tiles, 13 x 25 x 1 N tiles x 1 images = 325 tiles, 2.5 per CTA
    Entry('conv1x1_s1_256_128_n1_200x200', (1, 200, 200, 200, 200, 256, 0, 128, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 256, 1, 1), None, None, (1, 200, 200, 256), None, False, (1,),
          (('detector_256', 10), ('detector_512', 10),)),
    # N tile 128, 16x8 tiles, 7 x 13 x 1 N tiles x 1 images = 91 tiles, 1.0 per CTA
    Entry('conv3x3_s2_128_128_n1_100x100', (1, 200, 200, 100, 100, 128, 0, 128, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 128, 3, 3), None, None, (1, 200, 200, 128), None, False, (1,),
          (('detector_256', 11), ('detector_512', 11),)),
    # N tile 128, 16x8 tiles, 7 x 13 x 4 N tiles x 1 images = 364 tiles, 2.8 per CTA
    Entry('conv1x1_s1_128_512_n1_100x100', (1, 100, 100, 100, 100, 128, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 128, 1, 1), None, None, (1, 100, 100, 128), None, False, (1,),
          (('detector_256', 12), ('detector_256', 16), ('detector_256', 19), ('detector_256', 22), ('detector_512', 12), ('detector_512', 16), ('detector_512', 19), ('detector_512', 22),)),
    # N tile 128, 16x8 tiles, 7 x 13 x 4 N tiles x 1 images = 364 tiles, 2.8 per CTA
    Entry('conv1x1_s2_256_512_n1_100x100', (1, 200, 200, 100, 100, 256, 0, 512, 1, 1, 2, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 256, 1, 1), None, None, (1, 200, 200, 256), None, False, (1,),
          (('detector_256', 13), ('detector_512', 13),)),
    # N tile 128, 16x8 tiles, 7 x 13 x 1 N tiles x 1 images = 91 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_128_n1_100x100', (1, 100, 100, 100, 100, 512, 0, 128, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 512, 1, 1), None, None, (1, 100, 100, 512), None, False, (1,),
          (('detector_256', 14), ('detector_256', 17), ('detector_256', 20), ('detector_512', 14), ('detector_512', 17), ('detector_512', 20),)),
    # N tile 128, 16x8 tiles, 7 x 13 x 1 N tiles x 1 images = 91 tiles, 1.0 per CTA
    Entry('conv3x3_s1_128_128_n1_100x100', (1, 100, 100, 100, 100, 128, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (128, 128, 3, 3), None, None, (1, 100, 100, 128), None, False, (1,),
          (('detector_256', 15), ('detector_256', 18), ('detector_256', 21), ('detector_512', 15), ('detector_512', 18), ('detector_512', 21),)),
    # N tile 128, 16x8 tiles, 7 x 13 x 2 N tiles x 1 images = 182 tiles, 1.4 per CTA
    Entry('conv1x1_s1_512_256_n1_100x100', (1, 100, 100, 100, 100, 512, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 512, 1, 1), None, None, (1, 100, 100, 512), None, False, (1,),
          (('detector_256', 23), ('detector_256', 56), ('detector_512', 23), ('detector_512', 56),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 2 N tiles x 1 images = 56 tiles, 1.0 per CTA
    Entry('conv3x3_s2_256_256_n1_50x50', (1, 100, 100, 50, 50, 256, 0, 256, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 100, 100, 256), None, False, (1,),
          (('detector_256', 24), ('detector_512', 24),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 8 N tiles x 1 images = 224 tiles, 1.7 per CTA
    Entry('conv1x1_s1_256_1024_n1_50x50', (1, 50, 50, 50, 50, 256, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 256, 1, 1), None, None, (1, 50, 50, 256), None, False, (1,),
          (('detector_256', 25), ('detector_256', 29), ('detector_256', 32), ('detector_256', 35), ('detector_256', 38), ('detector_256', 41), ('detector_512', 25), ('detector_512', 29), ('detector_512', 32), ('detector_512', 35), ('detector_512', 38), ('detector_512', 41),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 8 N tiles x 1 images = 224 tiles, 1.7 per CTA
    Entry('conv1x1_s2_512_1024_n1_50x50', (1, 100, 100, 50, 50, 512, 0, 1024, 1, 1, 2, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 512, 1, 1), None, None, (1, 100, 100, 512), None, False, (1,),
          (('detector_256', 26), ('detector_512', 26),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 2 N tiles x 1 images = 56 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_256_n1_50x50', (1, 50, 50, 50, 50, 1024, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 1024, 1, 1), None, None, (1, 50, 50, 1024), None, False, (1,),
          (('detector_256', 27), ('detector_256', 30), ('detector_256', 33), ('detector_256', 36), ('detector_256', 39), ('detector_256', 54), ('detector_512', 27), ('detector_512', 30), ('detector_512', 33), ('detector_512', 36), ('detector_512', 39), ('detector_512', 54),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 2 N tiles x 1 images = 56 tiles, 1.0 per CTA
    Entry('conv3x3_s1_256_256_n1_50x50', (1, 50, 50, 50, 50, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 50, 50, 256), None, False, (1,),
          (('detector_256', 28), ('detector_256', 31), ('detector_256', 34), ('detector_256', 37), ('detector_256', 40), ('detector_256', 55), ('detector_256', 64), ('detector_512', 28), ('detector_512', 31), ('detector_512', 34), ('detector_512', 37), ('detector_512', 40), ('detector_512', 55), ('detector_512', 64),)),
    # N tile 128, 16x8 tiles, 4 x 7 x 4 N tiles x 1 images = 112 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_512_n1_50x50', (1, 50, 50, 50, 50, 1024, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 1024, 1, 1), None, None, (1, 50, 50, 1024), None, False, (1,),
          (('detector_256', 42), ('detector_512', 42),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv3x3_s2_512_512_n1_25x25', (1, 50, 50, 25, 25, 512, 0, 512, 3, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (1, 50, 50, 512), None, False, (1,),
          (('detector_256', 43), ('detector_512', 43),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 16 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv1x1_s1_512_2048_n1_25x25', (1, 25, 25, 25, 25, 512, 0, 2048, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (2048, 512, 1, 1), None, None, (1, 25, 25, 512), None, False, (1,),
          (('detector_256', 44), ('detector_256', 48), ('detector_256', 51), ('detector_512', 44), ('detector_512', 48), ('detector_512', 51),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 16 N tiles x 1 images = 128 tiles, 1.0 per CTA
    Entry('conv1x1_s2_1024_2048_n1_25x25', (1, 50, 50, 25, 25, 1024, 0, 2048, 1, 1, 2, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (2048, 1024, 1, 1), None, None, (1, 50, 50, 1024), None, False, (1,),
          (('detector_256', 45), ('detector_512', 45),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv1x1_s1_2048_512_n1_25x25', (1, 25, 25, 25, 25, 2048, 0, 512, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 2048, 1, 1), None, None, (1, 25, 25, 2048), None, False, (1,),
          (('detector_256', 46), ('detector_256', 49), ('detector_512', 46), ('detector_512', 49),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 4 N tiles x 1 images = 32 tiles, 1.0 per CTA
    Entry('conv3x3_s1_512_512_n1_25x25', (1, 25, 25, 25, 25, 512, 0, 512, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (512, 512, 3, 3), None, None, (1, 25, 25, 512), None, False, (1,),
          (('detector_256', 47), ('detector_256', 50), ('detector_512', 47), ('detector_512', 50),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 2 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('conv1x1_s1_2048_256_n1_25x25', (1, 25, 25, 25, 25, 2048, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 2048, 1, 1), None, None, (1, 25, 25, 2048), None, False, (1,),
          (('detector_256', 52), ('detector_512', 52),)),
    # N tile 128, 16x8 tiles, 2 x 4 x 2 N tiles x 1 images = 16 tiles, 1.0 per CTA
    Entry('conv3x3_s1_256_256_n1_25x25', (1, 25, 25, 25, 25, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 25, 25, 256), None, False, (1,),
          (('detector_256', 53), ('detector_256', 66), ('detector_512', 53), ('detector_512', 66),)),
    # N tile 128, 16x8 tiles, 7 x 13 x 2 N tiles x 1 images = 182 tiles, 1.4 per CTA
    Entry('conv3x3_s1_256_256_n1_100x100', (1, 100, 100, 100, 100, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 100, 100, 256), None, False, (1,),
          (('detector_256', 57), ('detector_256', 62), ('detector_512', 57), ('detector_512', 62),)),
    # N tile 128, 16x8 tiles, 13 x 25 x 2 N tiles x 1 images = 650 tiles, 4.9 per CTA
    Entry('conv1x1_s1_256_256_n1_200x200', (1, 200, 200, 200, 200, 256, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 1, 1), None, None, (1, 200, 200, 256), None, False, (1,),
          (('detector_256', 58), ('detector_512', 58),)),
    # N tile 128, 16x8 tiles, 13 x 25 x 2 N tiles x 1 images = 650 tiles, 4.9 per CTA
    Entry('conv3x3_s1_256_256_n1_200x200', (1, 200, 200, 200, 200, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 200, 200, 256), None, False, (1,),
          (('detector_256', 59), ('detector_256', 60), ('detector_512', 59), ('detector_512', 60),)),
    # N tile 16, 16x8 tiles, 13 x 25 x 1 N tiles x 1 images = 325 tiles, 2.5 per CTA
    Entry('conv1x1_s1_256_16_n1_200x200', (1, 200, 200, 200, 200, 256, 0, 16, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (16, 256, 1, 1), None, None, (1, 200, 200, 256), None, False, (1,),
          (('detector_256', 61), ('detector_512', 61),)),
    # N tile 16, 16x8 tiles, 7 x 13 x 1 N tiles x 1 images = 91 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_16_n1_100x100', (1, 100, 100, 100, 100, 256, 0, 16, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (16, 256, 1, 1), None, None, (1, 100, 100, 256), None, False, (1,),
          (('detector_256', 63), ('detector_512', 63),)),
    # N tile 16, 16x8 tiles, 4 x 7 x 1 N tiles x 1 images = 28 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_16_n1_50x50', (1, 50, 50, 50, 50, 256, 0, 16, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (16, 256, 1, 1), None, None, (1, 50, 50, 256), None, False, (1,),
          (('detector_256', 65), ('detector_512', 65),)),
    # N tile 16, 16x8 tiles, 2 x 4 x 1 N tiles x 1 images = 8 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_16_n1_25x25', (1, 25, 25, 25, 25, 256, 0, 16, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (16, 256, 1, 1), None, None, (1, 25, 25, 256), None, False, (1,),
          (('detector_256', 67), ('detector_512', 67),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 1 images = 4 tiles, 1.0 per CTA
    Entry('conv3x3_s1_256_256_n1_13x13', (1, 13, 13, 13, 13, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (1, 13, 13, 256), None, False, (1,),
          (('detector_256', 68), ('detector_512', 68),)),
    # N tile 16, 16x8 tiles, 1 x 2 x 1 N tiles x 1 images = 2 tiles, 1.0 per CTA
    Entry('conv1x1_s1_256_16_n1_13x13', (1, 13, 13, 13, 13, 256, 0, 16, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (16, 256, 1, 1), None, None, (1, 13, 13, 256), None, False, (1,),
          (('detector_256', 69), ('detector_512', 69),)),
    # N tile 128, 16x8 tiles, 8 x 1 x 8 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv1x1_s1_12544_1024_n1_125x8', (1, 125, 8, 125, 8, 12544, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 12544, 1, 1), None, None, (1, 125, 8, 12544), None, False, (1,),
          (('detector_256', 70), ('detector_512', 70),)),
    # N tile 128, 16x8 tiles, 8 x 1 x 8 N tiles x 1 images = 64 tiles, 1.0 per CTA
    Entry('conv1x1_s1_1024_1024_n1_125x8', (1, 125, 8, 125, 8, 1024, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 1024, 1, 1), None, None, (1, 125, 8, 1024), None, False, (1,),
          (('detector_256', 71), ('detector_512', 71),)),
    # N tile 16, 16x8 tiles, 8 x 1 x 29 N tiles x 1 images = 232 tiles, 1.8 per CTA
    Entry('conv1x1_s1_1024_464_n1_125x8', (1, 125, 8, 125, 8, 1024, 0, 464, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (464, 1024, 1, 1), None, None, (1, 125, 8, 1024), None, False, (1,),
          (('detector_256', 72), ('detector_512', 72),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 100 images = 400 tiles, 3.0 per CTA
    Entry('conv3x3_s1_256_256_n100_14x14', (100, 14, 14, 14, 14, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (100, 14, 14, 256), None, False, (1,),
          (('detector_256', 73), ('detector_256', 74), ('detector_256', 75), ('detector_256', 76), ('detector_512', 73), ('detector_512', 74), ('detector_512', 75), ('detector_512', 76),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 8 N tiles x 100 images = 1600 tiles, 12.1 per CTA
    Entry('conv1x1_s1_256_1024_n100_14x14', (100, 14, 14, 14, 14, 256, 0, 1024, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (1024, 256, 1, 1), None, None, (100, 14, 14, 256), None, False, (1,),
          (('detector_256', 77), ('detector_512', 77),)),
    # N tile 32, 16x8 tiles, 2 x 4 x 3 N tiles x 100 images = 2400 tiles, 18.2 per CTA
    Entry('conv1x1_s1_256_96_n100_28x28', (100, 28, 28, 28, 28, 256, 0, 96, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, -1),
          (96, 256, 1, 1), None, None, (100, 28, 28, 256), None, False, (1,),
          (('detector_256', 78), ('detector_512', 78),)),
    # N tile 64, 32x8 tiles, 1 x 4 x 3 N tiles x 64 images = 768 tiles, 5.8 per CTA
    Entry('conv5x5_s1_64_192_n64_31x31', (64, 31, 31, 31, 31, 64, 0, 192, 5, 5, 1, 2, 1, 0, 0, 0, 0, 0, 0, -1),
          (192, 64, 5, 5), None, None, (64, 31, 31, 64), None, False, (1,),
          (('lpips_b32_256', 0),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 3 N tiles x 64 images = 384 tiles, 2.9 per CTA
    Entry('conv3x3_s1_192_384_n64_15x15', (64, 15, 15, 15, 15, 192, 0, 384, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (384, 192, 3, 3), None, None, (64, 15, 15, 192), None, False, (1,),
          (('lpips_b32_256', 1),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 64 images = 256 tiles, 1.9 per CTA
    Entry('conv3x3_s1_384_256_n64_15x15', (64, 15, 15, 15, 15, 384, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 384, 3, 3), None, None, (64, 15, 15, 384), None, False, (1,),
          (('lpips_b32_256', 2),)),
    # N tile 128, 16x8 tiles, 1 x 2 x 2 N tiles x 64 images = 256 tiles, 1.9 per CTA
    Entry('conv3x3_s1_256_256_n64_15x15', (64, 15, 15, 15, 15, 256, 0, 256, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, -1),
          (256, 256, 3, 3), None, None, (64, 15, 15, 256), None, False, (1,),
          (('lpips_b32_256', 3),)),
    # N tile 64, 32x8 tiles, 5 x 19 x 1 N tiles x 32 images = 3040 tiles, 23.0 per CTA
    Entry('conv3x3_s1_64_64_n32_147x147_p0_pw0', (32, 149, 149, 147, 147, 64, 0, 64, 3, 3, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (32, 32, 3, 3), 64, 64, (32, 149, 149, 64), None, False, (1,),
          (('inception_b32_256', 0),)),
    # N tile 64, 32x8 tiles, 5 x 19 x 1 N tiles x 32 images = 3040 tiles, 23.0 per CTA
    Entry('conv3x3_s1_64_64_n32_147x147_pw1', (32, 147, 147, 147, 147, 64, 0, 64, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1),
          (64, 32, 3, 3), 64, 64, (32, 147, 147, 64), None, False, (1,),
          (('inception_b32_256', 1),)),
    # N tile 128, 16x8 tiles, 5 x 10 x 1 N tiles x 32 images = 1600 tiles, 12.1 per CTA
    Entry('conv1x1_s1_64_128_n32_73x73_pw0', (32, 73, 73, 73, 73, 64, 0, 128, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (80, 64, 1, 1), 128, 64, (32, 73, 73, 64), None, False, (1,),
          (('inception_b32_256', 2),)),
    # N tile 64, 32x8 tiles, 3 x 9 x 3 N tiles x 32 images = 2592 tiles, 19.6 per CTA
    Entry('conv3x3_s1_128_192_n32_71x71_p0_pw0', (32, 73, 73, 71, 71, 128, 0, 192, 3, 3, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (192, 80, 3, 3), 192, 128, (32, 73, 73, 128), None, False, (1,),
          (('inception_b32_256', 3),)),
    # N tile 128, 16x8 tiles, 3 x 5 x 2 N tiles x 32 images = 960 tiles, 7.3 per CTA
    Entry('conv1x1_s1_192_256_n32_35x35_pw0', (32, 35, 35, 35, 35, 192, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (208, 192, 1, 1), 256, 192, (32, 35, 35, 192), None, False, (1,),
          (('inception_b32_256', 4),)),
    # N tile 64, 32x8 tiles, 2 x 5 x 1 N tiles x 32 images = 320 tiles, 2.4 per CTA
    Entry('conv5x5_s1_64_64_n32_35x35_pw2', (32, 35, 35, 35, 35, 64, 0, 64, 5, 5, 1, 2, 1, 0, 0, 0, 0, 0, 0, 2),
          (64, 48, 5, 5), 64, 64, (32, 35, 35, 64), None, False, (1,),
          (('inception_b32_256', 5), ('inception_b32_256', 9), ('inception_b32_256', 13),)),
    # N tile 128, 16x8 tiles, 3 x 5 x 1 N tiles x 32 images = 480 tiles, 3.6 per CTA
    Entry('conv3x3_s1_64_128_n32_35x35_pw1', (32, 35, 35, 35, 35, 64, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1),
          (96, 64, 3, 3), 128, 64, (32, 35, 35, 64), None, False, (1,),
          (('inception_b32_256', 6), ('inception_b32_256', 10), ('inception_b32_256', 14), ('inception_b32_256', 18),)),
    # N tile 128, 16x8 tiles, 3 x 5 x 1 N tiles x 32 images = 480 tiles, 3.6 per CTA
    Entry('conv3x3_s1_128_128_n32_35x35_pw1', (32, 35, 35, 35, 35, 128, 0, 128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1),
          (96, 96, 3, 3), 128, 128, (32, 35, 35, 128), None, False, (1,),
          (('inception_b32_256', 7), ('inception_b32_256', 11), ('inception_b32_256', 15),)),
    # N tile 128, 16x8 tiles, 3 x 5 x 2 N tiles x 32 images = 960 tiles, 7.3 per CTA
    Entry('conv1x1_s1_256_256_n32_35x35_pw0', (32, 35, 35, 35, 35, 256, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (240, 256, 1, 1), 256, 256, (32, 35, 35, 256), None, False, (1,),
          (('inception_b32_256', 8),)),
    # N tile 128, 16x8 tiles, 3 x 5 x 2 N tiles x 32 images = 960 tiles, 7.3 per CTA
    Entry('conv1x1_s1_320_256_n32_35x35_pw0', (32, 35, 35, 35, 35, 320, 0, 256, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (240, 288, 1, 1), 256, 320, (32, 35, 35, 320), None, False, (1,),
          (('inception_b32_256', 12),)),
    # N tile 128, 16x8 tiles, 2 x 3 x 3 N tiles x 32 images = 576 tiles, 4.4 per CTA
    Entry('conv3x3_s2_320_384_n32_17x17_p0_pw0', (32, 35, 35, 17, 17, 320, 0, 384, 3, 3, 2, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (384, 288, 3, 3), 384, 320, (32, 35, 35, 320), None, False, (1,),
          (('inception_b32_256', 16),)),
    # N tile 64, 32x8 tiles, 2 x 5 x 1 N tiles x 32 images = 320 tiles, 2.4 per CTA
    Entry('conv1x1_s1_320_64_n32_35x35_pw0', (32, 35, 35, 35, 35, 320, 0, 64, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (64, 288, 1, 1), 64, 320, (32, 35, 35, 320), None, False, (1,),
          (('inception_b32_256', 17),)),
    # N tile 128, 16x8 tiles, 2 x 3 x 1 N tiles x 32 images = 192 tiles, 1.5 per CTA
    Entry('conv3x3_s2_128_128_n32_17x17_p0_pw0', (32, 35, 35, 17, 17, 128, 0, 128, 3, 3, 2, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (96, 96, 3, 3), 128, 128, (32, 35, 35, 128), None, False, (1,),
          (('inception_b32_256', 19),)),
    # N tile 128, 16x8 tiles, 2 x 3 x 5 N tiles x 32 images = 960 tiles, 7.3 per CTA
    Entry('conv1x1_s1_768_640_n32_17x17_pw0', (32, 17, 17, 17, 17, 768, 0, 640, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (640, 768, 1, 1), 640, 768, (32, 17, 17, 768), None, False, (1,),
          (('inception_b32_256', 20),)),
    # N tile 128, 16x8 tiles, 2 x 3 x 1 N tiles x 32 images = 192 tiles, 1.5 per CTA
    Entry('conv1x7_s1_128_128_n32_17x17_pw3', (32, 17, 17, 17, 17, 128, 0, 128, 1, 7, 1, 0, 1, 0, 0, 0, 0, 0, 0, 3),
          (128, 128, 1, 7), 128, 128, (32, 17, 17, 128), None, False, (1,),
          (('inception_b32_256', 21), ('inception_b32_256', 24),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv7x1_s1_128_192_n32_17x17_pw0', (32, 17, 17, 17, 17, 128, 0, 192, 7, 1, 1, 3, 1, 0, 0, 0, 0, 0, 0, 0),
          (192, 128, 7, 1), 192, 128, (32, 17, 17, 128), None, False, (1,),
          (('inception_b32_256', 22),)),
    # N tile 128, 16x8 tiles, 2 x 3 x 1 N tiles x 32 images = 192 tiles, 1.5 per CTA
    Entry('conv7x1_s1_128_128_n32_17x17_pw0', (32, 17, 17, 17, 17, 128, 0, 128, 7, 1, 1, 3, 1, 0, 0, 0, 0, 0, 0, 0),
          (128, 128, 7, 1), 128, 128, (32, 17, 17, 128), None, False, (1,),
          (('inception_b32_256', 23), ('inception_b32_256', 25),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv1x7_s1_128_192_n32_17x17_pw3', (32, 17, 17, 17, 17, 128, 0, 192, 1, 7, 1, 0, 1, 0, 0, 0, 0, 0, 0, 3),
          (192, 128, 1, 7), 192, 128, (32, 17, 17, 128), None, False, (1,),
          (('inception_b32_256', 26),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 11 N tiles x 32 images = 1056 tiles, 8.0 per CTA
    Entry('conv1x1_s1_768_704_n32_17x17_pw0', (32, 17, 17, 17, 17, 768, 0, 704, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (704, 768, 1, 1), 704, 768, (32, 17, 17, 768), None, False, (1,),
          (('inception_b32_256', 27), ('inception_b32_256', 34),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv1x7_s1_192_192_n32_17x17_pw3_v1', (32, 17, 17, 17, 17, 192, 0, 192, 1, 7, 1, 0, 1, 0, 0, 0, 0, 0, 0, 3),
          (160, 160, 1, 7), 192, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 28), ('inception_b32_256', 31), ('inception_b32_256', 35), ('inception_b32_256', 38),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv7x1_s1_192_192_n32_17x17_pw0_v1', (32, 17, 17, 17, 17, 192, 0, 192, 7, 1, 1, 3, 1, 0, 0, 0, 0, 0, 0, 0),
          (192, 160, 7, 1), 192, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 29), ('inception_b32_256', 36),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv7x1_s1_192_192_n32_17x17_pw0_v2', (32, 17, 17, 17, 17, 192, 0, 192, 7, 1, 1, 3, 1, 0, 0, 0, 0, 0, 0, 0),
          (160, 160, 7, 1), 192, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 30), ('inception_b32_256', 32), ('inception_b32_256', 37), ('inception_b32_256', 39),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv1x7_s1_192_192_n32_17x17_pw3_v2', (32, 17, 17, 17, 17, 192, 0, 192, 1, 7, 1, 0, 1, 0, 0, 0, 0, 0, 0, 3),
          (192, 160, 1, 7), 192, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 33), ('inception_b32_256', 40),)),
    # N tile 128, 16x8 tiles, 2 x 3 x 6 N tiles x 32 images = 1152 tiles, 8.7 per CTA
    Entry('conv1x1_s1_768_768_n32_17x17_pw0', (32, 17, 17, 17, 17, 768, 0, 768, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (768, 768, 1, 1), 768, 768, (32, 17, 17, 768), None, False, (1,),
          (('inception_b32_256', 41),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv1x7_s1_192_192_n32_17x17_pw3_v3', (32, 17, 17, 17, 17, 192, 0, 192, 1, 7, 1, 0, 1, 0, 0, 0, 0, 0, 0, 3),
          (192, 192, 1, 7), 192, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 42), ('inception_b32_256', 45), ('inception_b32_256', 47), ('inception_b32_256', 50),)),
    # N tile 64, 32x8 tiles, 1 x 3 x 3 N tiles x 32 images = 288 tiles, 2.2 per CTA
    Entry('conv7x1_s1_192_192_n32_17x17_pw0_v3', (32, 17, 17, 17, 17, 192, 0, 192, 7, 1, 1, 3, 1, 0, 0, 0, 0, 0, 0, 0),
          (192, 192, 7, 1), 192, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 43), ('inception_b32_256', 44), ('inception_b32_256', 46), ('inception_b32_256', 51),)),
    # N tile 128, 16x8 tiles, 2 x 3 x 3 N tiles x 32 images = 576 tiles, 4.4 per CTA
    Entry('conv1x1_s1_768_384_n32_17x17_pw0', (32, 17, 17, 17, 17, 768, 0, 384, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (384, 768, 1, 1), 384, 768, (32, 17, 17, 768), None, False, (1,),
          (('inception_b32_256', 48),)),
    # N tile 64, 32x8 tiles, 1 x 1 x 5 N tiles x 32 images = 160 tiles, 1.2 per CTA
    Entry('conv3x3_s2_192_320_n32_8x8_p0_pw0', (32, 17, 17, 8, 8, 192, 0, 320, 3, 3, 2, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (320, 192, 3, 3), 320, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 49),)),
    # N tile 64, 32x8 tiles, 1 x 1 x 3 N tiles x 32 images = 96 tiles, 1.0 per CTA
    Entry('conv3x3_s2_192_192_n32_8x8_p0_pw0', (32, 17, 17, 8, 8, 192, 0, 192, 3, 3, 2, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (192, 192, 3, 3), 192, 192, (32, 17, 17, 192), None, False, (1,),
          (('inception_b32_256', 52),)),
    # N tile 64, 32x8 tiles, 1 x 1 x 21 N tiles x 32 images = 672 tiles, 5.1 per CTA
    Entry('conv1x1_s1_1280_1344_n32_8x8_pw0', (32, 8, 8, 8, 8, 1280, 0, 1344, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (1344, 1280, 1, 1), 1344, 1280, (32, 8, 8, 1280), None, False, (1,),
          (('inception_b32_256', 53),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 3 N tiles x 32 images = 96 tiles, 1.0 per CTA
    Entry('conv3x3_s1_448_384_n32_8x8_pw1', (32, 8, 8, 8, 8, 448, 0, 384, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0, 0, 1),
          (384, 448, 3, 3), 384, 448, (32, 8, 8, 448), None, False, (1,),
          (('inception_b32_256', 54), ('inception_b32_256', 60),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 3 N tiles x 32 images = 96 tiles, 1.0 per CTA
    Entry('conv1x3_s1_384_384_n32_8x8_pw1', (32, 8, 8, 8, 8, 384, 0, 384, 1, 3, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1),
          (384, 384, 1, 3), 384, 384, (32, 8, 8, 384), None, False, (1,),
          (('inception_b32_256', 55), ('inception_b32_256', 57), ('inception_b32_256', 61), ('inception_b32_256', 63),)),
    # N tile 128, 16x8 tiles, 1 x 1 x 3 N tiles x 32 images = 96 tiles, 1.0 per CTA
    Entry('conv3x1_s1_384_384_n32_8x8_pw0', (32, 8, 8, 8, 8, 384, 0, 384, 3, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0),
          (384, 384, 3, 1), 384, 384, (32, 8, 8, 384), None, False, (1,),
          (('inception_b32_256', 56), ('inception_b32_256', 58), ('inception_b32_256', 62), ('inception_b32_256', 64),)),
    # N tile 64, 32x8 tiles, 1 x 1 x 21 N tiles x 32 images = 672 tiles, 5.1 per CTA
    Entry('conv1x1_s1_2048_1344_n32_8x8_pw0', (32, 8, 8, 8, 8, 2048, 0, 1344, 1, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0),
          (1344, 2048, 1, 1), 1344, 2048, (32, 8, 8, 2048), None, False, (1,),
          (('inception_b32_256', 59),)),
]
