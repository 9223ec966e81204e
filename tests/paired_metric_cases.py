"""Float64 contract cases of the paired-metric kernels (csrc/metrics.cu), shared by test_paired_metrics_cpu.py and
test_paired_metrics_gpu.py:

  * ``ssim_psnr_ref``: SSIM and PSNR as skimage 0.16.2 defines them (oracle/metrics_ref.py documents the definition),
    at a precision far below the bars.  Every 7x7 window sum is taken directly, as the sum of seven horizontal sums of
    seven terms, in np.longdouble (64-bit mantissa): x * y of float32 inputs is exact there, and so are the moments to
    ~1e-19.  scipy's uniform_filter keeps running sums that drift along a row, so the oracle does not serve here.  The
    PSNR squared errors are float32, as numpy computes them, and are summed exactly (math.fsum per frame).
  * ``restated``: k_ssim_tiles + k_ssim_finish in float64 numpy, tile by tile: the 14 x 70 input window of each 8 x 64
    tile with its 3-pixel halo (0 outside the image), horizontal then vertical 7-sums, the map over the tile's pixels
    that are 3 or more from every border, and the per-tile partials (map sum, squared-error sum, min(ref)) that the
    finish pass reduces per frame.  ``MUTANTS`` are plausible kernel bugs; each must exceed a bar at least 4x on a case.
  * ``CASES``: (n, h, w, from01, content, seed), one per edge of ``REQUIRED_EDGES``: partial tiles in x and y, the
    smallest frame, the crop inside a partial tile, the PSNR data range decided in the last partial tile, NaN / inf
    isolation, and a batch past the 21845 frames one launch's grid.z holds.
  * ``LPIPS_CASES``: the sizes where AlexNet's features shrink to 1 x 1 .. 3 x 3, and where floor- and ceil-mode pools
    differ.

Frames are [n,3,h,w] float32, in [0,1] when from01 (mapped by x * 2 - 1 in float32) and in [-1,1] otherwise.
"""
import collections
import math

import numpy as np
import torch
from scipy.ndimage import uniform_filter

from oracle import metrics_ref as R

SSIM_BAR, PSNR_BAR, LPIPS_BAR = 1e-12, 1e-10, 1e-6       # per frame; LPIPS also per layer term
TILE_H, TILE_W, CROP = 8, 64, 3
WIN_H, WIN_W = TILE_H + 2 * CROP, TILE_W + 2 * CROP
K1, K2, DATA_RANGE = 0.01, 0.03, 2.0
MAX_FRAMES_PER_LAUNCH = 65535 // 3

Case = collections.namedtuple("Case", "edge n h w from01 content seed")

CASES = [
    # sizes: one interior pixel, one row / column of tiles, one full tile and one past it, partial tiles both ways
    Case("7x7", 3, 7, 7, 1, "noise", 21),
    Case("7x200", 1, 7, 200, 0, "smooth", 22),
    Case("200x7", 1, 200, 7, 1, "smooth", 23),
    Case("8x64", 1, 8, 64, 0, "noise", 24),
    Case("9x65", 3, 9, 65, 1, "smooth", 25),
    Case("15x63", 5, 15, 63, 0, "smooth", 26),
    Case("16x128", 1, 16, 128, 1, "noise", 27),
    Case("17x129", 3, 17, 129, 0, "smooth", 28),
    Case("14x70_crop_in_second_column_tile", 3, 14, 70, 1, "border", 29),
    Case("71x71", 1, 71, 71, 0, "smooth", 30),
    Case("333x517", 1, 333, 517, 1, "smooth", 31),
    Case("480x640", 1, 480, 640, 0, "smooth", 32),
    Case("256x256", 3, 256, 256, 1, "smooth", 33),
    Case("512x512", 1, 512, 512, 0, "smooth", 34),
    # batch: more frames than one launch's grid.z holds
    Case("batch_21846_frames", MAX_FRAMES_PER_LAUNCH + 1, 7, 7, 1, "noise", 35),
    # content
    Case("full_range_noise", 3, 71, 71, 1, "noise", 36),
    Case("bright_flat", 3, 17, 129, 0, "flat", 37),
    Case("constant", 3, 9, 65, 1, "constant", 38),
    Case("identical", 3, 15, 63, 0, "identical", 39),
    Case("strong_border", 3, 33, 135, 0, "border", 40),
    Case("tile_boundary_pixels", 3, 17, 129, 0, "tile_pixels", 41),
    Case("last_pixel_of_last_tile", 1, 17, 129, 1, "last_pixel", 42),
    # PSNR data range: min(ref) only in the last partial tile of channel 2 of the last frame
    Case("range_min_zero", 3, 17, 129, 0, "min_zero", 43),
    Case("range_min_minus_2^-24", 3, 17, 129, 0, "min_neg_ulp", 44),
    Case("range_min_negative_zero", 3, 17, 129, 0, "min_neg_zero", 45),
    Case("range_min_minus_2^-24_from01", 3, 9, 65, 1, "min_neg_ulp", 46),
    # isolation: NaN in frame 1's pred, +inf in frame 3's
    Case("nan_inf_isolation", 5, 17, 129, 1, "nan_inf", 47),
]
REQUIRED_EDGES = [
    "7x7", "7x200", "200x7", "8x64", "9x65", "15x63", "16x128", "17x129", "14x70_crop_in_second_column_tile", "71x71",
    "333x517", "480x640", "256x256", "512x512", "batch_21846_frames",
    "full_range_noise", "bright_flat", "constant", "identical", "strong_border", "tile_boundary_pixels",
    "last_pixel_of_last_tile",
    "range_min_zero", "range_min_minus_2^-24", "range_min_negative_zero", "range_min_minus_2^-24_from01",
    "nan_inf_isolation",
]
RANGE_MIN = {"min_zero": 0.0, "min_neg_ulp": -2.0 ** -24, "min_neg_zero": -0.0}
# (frame, channel, y, x) of the one-pixel differences: tile-boundary pixels x = 63 / 64, y = 7 / 8
TILE_PIXELS = ((0, 0, 7, 63), (1, 1, 8, 64), (2, 2, 7, 64), (2, 0, 8, 63))
NAN_AT, INF_AT = (1, 1, 8, 64), (3, 0, 7, 63)


def by_edge(edge):
    return next(c for c in CASES if c.edge == edge)


def _smooth01(rng, n, h, w):
    """Smooth frames with noise in [0,1], as metrics_cases makes them: 8x8 blocks, a 9x9 box filter, +-0.1 noise."""
    low = rng.random((n, 3, -(-h // 8), -(-w // 8)), dtype=np.float32)
    up = np.repeat(np.repeat(low, 8, axis=2), 8, axis=3)[:, :, :h, :w].astype(np.float64)
    ref = uniform_filter(up, size=(1, 1, 9, 9)).astype(np.float32)
    noise = (rng.random(ref.shape, dtype=np.float32) - np.float32(0.5)) * np.float32(0.2)
    return np.clip(ref + noise, 0, 1).astype(np.float32), ref


def _to_input(x01, from01):
    """[0,1] frames -> the kernel's input: unchanged with from01, else x * 2 - 1 in float32 (values stay in [-1,1])."""
    x01 = np.asarray(x01, np.float32)
    return x01 if from01 else (x01 * np.float32(2) - np.float32(1)).astype(np.float32)


def _from_unit(v, from01):
    """The input value that from01's x * 2 - 1 maps to v exactly (v itself without from01)."""
    if not from01:
        return np.float32(v)
    x = np.float32((v + 1.0) / 2.0)
    y = x * np.float32(2) - np.float32(1)
    assert y == np.float32(v) and np.signbit(y) == np.signbit(v), "x * 2 - 1 cannot give %r" % v
    return x


def make(case, clean=False):
    """-> (pred, ref) float32 [n,3,h,w], the kernel's input.  clean: the isolation case without its bad pixels."""
    n, h, w, from01, content = case.n, case.h, case.w, case.from01, case.content
    rng = np.random.default_rng(case.seed)
    if content == "noise":                                         # full range, independent
        p01, r01 = rng.random((n, 3, h, w), dtype=np.float32), rng.random((n, 3, h, w), dtype=np.float32)
    elif content == "flat":                                        # 0.95 +- 0.002 in [-1,1]
        p01, r01 = (np.float32(0.975) + (rng.random((2, n, 3, h, w), dtype=np.float32) - np.float32(0.5))
                    * np.float32(0.002)).astype(np.float32)
    elif content == "constant":
        p01 = np.broadcast_to(rng.random((n, 3, 1, 1), dtype=np.float32), (n, 3, h, w)).copy()
        r01 = np.broadcast_to(rng.random((n, 3, 1, 1), dtype=np.float32), (n, 3, h, w)).copy()
    elif content == "border":                                      # smooth, full-range noise in the 3-pixel border
        p01, r01 = _smooth01(rng, n, h, w)
        edge = np.ones((h, w), bool)
        edge[CROP:h - CROP, CROP:w - CROP] = False
        for a in (p01, r01):
            a[..., edge] = rng.random((n, 3, int(edge.sum())), dtype=np.float32)
    elif content in ("min_zero", "min_neg_ulp", "min_neg_zero"):  # ref >= 0.1 except one pixel
        p01, r01 = _smooth01(rng, n, h, w)
        r01 = (np.float32(0.55) + np.float32(0.45) * r01).astype(np.float32)
    else:                                                          # smooth, identical, one-pixel changes, nan_inf
        p01, r01 = _smooth01(rng, n, h, w)
    pred, ref = _to_input(p01, from01), _to_input(r01, from01)
    if content == "identical":
        pred = ref.copy()
    elif content in ("tile_pixels", "last_pixel"):
        pred = ref.copy()
        for img, ch, y, x in (TILE_PIXELS if content == "tile_pixels" else ((n - 1, 2, h - 1, w - 1),)):
            pred[img, ch, y, x] = _from_unit(0.5 if ref[img, ch, y, x] < _from_unit(0.0, from01) else -0.5, from01)
    elif content in RANGE_MIN:
        ref[n - 1, 2, h - 1, w - 1] = _from_unit(RANGE_MIN[content], from01)
    elif content == "nan_inf" and not clean:
        pred[NAN_AT], pred[INF_AT] = np.nan, np.inf
    return np.ascontiguousarray(pred), np.ascontiguousarray(ref)


def preprocess(x, from01):
    """from01's x * 2 - 1 in float32, as k_ssim_tiles' load (and the metrics' preprocess) computes it."""
    x = np.asarray(x, np.float32)
    return (x * np.float32(2) - np.float32(1)).astype(np.float32) if from01 else x


# ---- reference -----------------------------------------------------------------------------------------------------
assert np.finfo(np.longdouble).nmant >= 63, "the SSIM reference needs an 80-bit long double"


def _box7(a):
    """7x7 window sums of [..., h, w] -> [..., h-6, w-6]: each the sum of seven horizontal sums of seven terms."""
    hs = sum(a[..., :, k:a.shape[-1] - 6 + k] for k in range(7))
    return sum(hs[..., k:hs.shape[-2] - 6 + k, :] for k in range(7))


def ssim_psnr_ref(pred, ref, from01):
    """Per-frame (SSIM, PSNR) float64 [n] of skimage 0.16.2's structural_similarity(pred, ref, multichannel=True) and
    peak_signal_noise_ratio(image_true=ref, image_test=pred) on the [-1,1] images."""
    x32, y32 = preprocess(pred, from01), preprocess(ref, from01)
    L = np.longdouble
    x, y = x32.astype(L), y32.astype(L)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        mx, my = _box7(x) / 49, _box7(y) / 49
        mxx, myy, mxy = _box7(x * x) / 49, _box7(y * y) / 49, _box7(x * y) / 49
        cov = L(49) / L(48)
        vx, vy, vxy = cov * (mxx - mx * mx), cov * (myy - my * my), cov * (mxy - mx * my)
        c1, c2 = L((K1 * DATA_RANGE) ** 2), L((K2 * DATA_RANGE) ** 2)
        S = ((2 * mx * my + c1) * (2 * vxy + c2)) / ((mx * mx + my * my + c1) * (vx + vy + c2))
        ssim = S.mean(axis=(-2, -1)).mean(axis=-1).astype(np.float64)
        sq = ((y32 - x32) * (y32 - x32)).astype(np.float32).reshape(len(x32), -1)
        err = np.array([math.fsum(row.tolist()) for row in sq])
        mse = err / sq.shape[1]
        rng = np.where(y32.reshape(len(y32), -1).min(axis=1) >= 0, 1.0, 2.0)
        psnr = 10 * np.log10(rng * rng / mse)
    return ssim, psnr


def oracle_scores(pred, ref, from01, frames=None):
    """oracle/metrics_ref.py's per-frame SSIM and PSNR on the [-1,1] HWC images (frames: the indices to score)."""
    x, y = preprocess(pred, from01), preprocess(ref, from01)
    idx = range(len(x)) if frames is None else frames
    hwc = lambda a: np.transpose(a, (1, 2, 0))
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        s = np.array([R.structural_similarity(hwc(x[i]), hwc(y[i])) for i in idx])
        p = np.array([R.peak_signal_noise_ratio(image_true=hwc(y[i]), image_test=hwc(x[i])) for i in idx])
    return s, p


def err_over_bar(got, want, bar):
    """Per-frame |got - want| / bar; 0 where both are the same NaN or infinity, inf where only one is not finite."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    fin = np.isfinite(got) & np.isfinite(want)
    same = (np.isnan(got) & np.isnan(want)) | (np.isinf(got) & (got == want))
    r = np.where(same, 0.0, np.inf)
    r[fin] = np.abs(got[fin] - want[fin]) / bar
    return r


# ---- restatement of k_ssim_tiles + k_ssim_finish -------------------------------------------------------------------
MUTANTS = ["f32_moments", "population_covariance", "crop_2", "crop_4", "zero_halo", "drop_partial_col_tile",
           "drop_partial_row_tile", "min_over_interior", "min_channel0_only", "mse_interior_count", "from01_pred_only",
           "plane_order"]


def restated(pred, ref, from01, mutant=None):
    """k_ssim_tiles + k_ssim_finish in numpy -> per-frame (SSIM, PSNR) float64 [n].  mutant: None or one of MUTANTS:
      f32_moments            window sums and the map in float32;
      population_covariance  no 49/48;
      crop_2, crop_4         the map cropped by 2 or 4 pixels per side instead of 3;
      zero_halo              each tile's halo pixels from its neighbour tiles read as 0;
      drop_partial_col_tile  tiles past the right border contribute nothing; drop_partial_row_tile the same for rows;
      min_over_interior      min(ref) over the SSIM crop only; min_channel0_only over channel 0 only;
      mse_interior_count     the squared errors divided by 3 (h-6) (w-6);
      from01_pred_only       x * 2 - 1 applied to pred only;
      plane_order            frame i, channel c read from plane c * n + i instead of i * 3 + c."""
    n, _, h, w = pred.shape
    x = preprocess(pred, from01)
    y = preprocess(ref, from01 and mutant != "from01_pred_only")
    if mutant == "plane_order":
        x, y = (a.reshape(3, n, h, w).transpose(1, 0, 2, 3) for a in (x, y))
    gy, gx = -(-h // TILE_H), -(-w // TILE_W)
    pads = []
    for a in (x, y):                                               # the image in a zero frame of 3 + tile rounding
        p = np.zeros((n, 3, gy * TILE_H + 2 * CROP, gx * TILE_W + 2 * CROP), np.float32)
        p[..., CROP:CROP + h, CROP:CROP + w] = a
        # [n, 3, gy, gx, 14, 70]: the input window each tile loads
        win = np.lib.stride_tricks.sliding_window_view(p, (WIN_H, WIN_W), axis=(2, 3))
        pads.append(win[:, :, ::TILE_H, ::TILE_W].copy())
    wx, wy = pads
    if mutant == "zero_halo":
        for a in (wx, wy):
            a[..., :CROP, :] = a[..., -CROP:, :] = 0
            a[..., :, :CROP] = a[..., :, -CROP:] = 0
    dt = np.float32 if mutant == "f32_moments" else np.float64
    crop = {"crop_2": 2, "crop_4": 4}.get(mutant, CROP)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        a, b = wx.astype(dt), wy.astype(dt)
        m = []
        for q in (a, b, a * a, b * b, a * b):
            hs = q[..., 0:TILE_W]
            for k in range(1, 7):                                   # horizontal 7-sums, in order
                hs = hs + q[..., k:k + TILE_W]
            vs = hs[..., 0:TILE_H, :]
            for k in range(1, 7):                                   # vertical 7-sums, in order
                vs = vs + hs[..., k:k + TILE_H, :]
            m.append(vs / dt(49))
        ux, uy, uxx, uyy, uxy = m
        cov = dt(1) if mutant == "population_covariance" else dt(49) / dt(48)
        vx, vy, vxy = cov * (uxx - ux * ux), cov * (uyy - uy * uy), cov * (uxy - ux * uy)
        c1, c2 = dt((K1 * DATA_RANGE) ** 2), dt((K2 * DATA_RANGE) ** 2)
        S = ((2 * ux * uy + c1) * (2 * vxy + c2)) / ((ux * ux + uy * uy + c1) * (vx + vy + c2))
        # pixel coordinates of each tile position
        yy = (np.arange(gy)[:, None, None, None] * TILE_H + np.arange(TILE_H)[None, None, :, None])
        xx = (np.arange(gx)[None, :, None, None] * TILE_W + np.arange(TILE_W)[None, None, None, :])
        inside = (yy < h) & (xx < w)
        interior = inside & (yy >= crop) & (yy < h - crop) & (xx >= crop) & (xx < w - crop)
        keep = np.ones((gy, gx, 1, 1), bool)
        if mutant == "drop_partial_col_tile":
            keep &= (np.arange(gx) * TILE_W + TILE_W <= w)[None, :, None, None]
        if mutant == "drop_partial_row_tile":
            keep &= (np.arange(gy) * TILE_H + TILE_H <= h)[:, None, None, None]
        inside, interior = inside & keep, interior & keep
        s_part = np.where(interior, S, 0).astype(np.float64).sum(axis=(-2, -1))          # [n, 3, gy, gx]
        xc, yc = wx[..., CROP:CROP + TILE_H, CROP:CROP + TILE_W], wy[..., CROP:CROP + TILE_H, CROP:CROP + TILE_W]
        d = (yc - xc).astype(np.float32)
        e_part = np.where(inside, (d * d).astype(np.float32), 0).astype(np.float64).sum(axis=(-2, -1))
        min_mask = interior if mutant == "min_over_interior" else inside
        r_part = np.where(min_mask, yc, np.float32(np.inf)).min(axis=(-2, -1))
        ssim_c = s_part.sum(axis=(-2, -1)) / (float(h - 2 * crop) * float(w - 2 * crop))   # [n, 3]
        ssim = (ssim_c[:, 0] + ssim_c[:, 1] + ssim_c[:, 2]) / 3.0
        err = e_part.sum(axis=(1, 2, 3))
        count = 3.0 * (h - 2 * CROP) * (w - 2 * CROP) if mutant == "mse_interior_count" else 3.0 * h * w
        mse = err / count
        rmin = (r_part[:, :1] if mutant == "min_channel0_only" else r_part).min(axis=(1, 2, 3)).astype(np.float64)
        rng = np.where(rmin >= 0, 1.0, 2.0)
        psnr = 10.0 * np.log10(rng * rng / mse)
    return ssim, psnr


# ---- LPIPS ---------------------------------------------------------------------------------------------------------
LpipsCase = collections.namedtuple("LpipsCase", "edge n h w from01 seed")
LPIPS_CASES = [
    LpipsCase("31x31_last_pool_1x1", 1, 31, 31, 1, 51),              # conv1 7, pool1 3, pool2 1: k_lpips_layer hw = 1
    LpipsCase("43x43_floor_differs_from_ceil", 2, 43, 43, 0, 52),    # conv1 10, pool1 4 (ceil 5), pool2 1 (ceil 2)
    LpipsCase("37x90_non_square", 2, 37, 90, 1, 53),
    LpipsCase("333x517", 1, 333, 517, 0, 54),
    LpipsCase("batch33_43x61", 33, 43, 61, 1, 55),                  # calculate_score's chunks of 32 and 1
]
LPIPS_REFUSED = (30, 30)                                          # pool1 gives 2 x 2: AlexNet's second pool cannot run


def make_lpips(case):
    p01, r01 = _smooth01(np.random.default_rng(case.seed), case.n, case.h, case.w)
    return _to_input(p01, case.from01), _to_input(r01, case.from01)


def lpips_ref(pred, ref, from01, convs, lins):
    """oracle.metrics_ref.lpips in float64 of the kernel's inputs -> (score [n], layers [n,5]) numpy."""
    p, r = (torch.from_numpy(preprocess(a, from01)) for a in (pred, ref))
    with torch.no_grad():
        val, layers = R.lpips(r, p, convs, lins, torch.float64)
    return val.numpy(), layers.numpy()
