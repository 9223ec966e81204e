"""CPU oracle of the input path (lwb_frames_in, kernels.frames_in): what cv2.resize(frame, (S, S)) computes on uint8 with
its default INTER_LINEAR, restated in numpy, and the cases both the CPU and the GPU tests sweep.

OpenCV's uint8 bilinear resize is fixed point, and its documentation does not say how.  What it computes:
  * per output coordinate d: scale = 1 / (S / src) in double, f = (float)((d + 0.5) * scale - 0.5), s = floor(f), f -= s
    (in float); the weights (1 - f) * 2048 and f * 2048 are each rounded half to even on their own.  Columns clamp their
    weights at the borders (s < 0 or s >= src - 1: f = 0, s into range); rows keep their weights and clamp only the row
    indices.
  * horizontal pass, exact in int32: H = p[s0] * a0 + p[s1] * a1.
  * vertical pass as its 16-bit vector code rounds it, for every output byte:
      ((H0 >> 4) * b0 >> 16) + ((H1 >> 4) * b1 >> 16) + 2 >> 2
    and not (H0 * b0 + H1 * b1 + 2^21) >> 22, which is off by one in about 20 000 bytes of a 256x256 frame.
Computing f in double instead of float is what made upscales (100x90 -> 256) differ in a few hundred bytes.
"""
import numpy as np

HMR_SIZE = 224

# (h, w, S): the ratios the Imitator meets (1024^2 and VGA frames to 256 / 224, upscales of small frames), degenerate
# sources (1x1, one row, one column), sources equal to the target, odd primes, exact 2x / 4x both ways, 512 targets, and
# targets that are not multiples of 16 (where OpenCV's scalar tail would round differently, were it used).
SWEEP = [
    (1024, 1024, 256), (1024, 1024, 224), (480, 640, 256), (333, 517, 224), (100, 90, 256), (256, 256, 224),
    (1, 1, 256), (1, 37, 224), (41, 1, 256), (1, 640, 256), (480, 1, 224),
    (256, 256, 256), (224, 224, 224), (512, 512, 512),
    (97, 131, 224), (331, 517, 256), (131, 97, 512),
    (512, 512, 256), (1024, 1024, 256), (128, 128, 256), (64, 64, 256), (128, 128, 512), (2048, 2048, 512),
    (720, 1280, 512), (1080, 1920, 256), (3, 5, 100), (50, 50, 97), (300, 200, 13),
]


def coefficients(src, dst, clamp):
    """Source indices (s0, s1) and fixed-point weights (a0, a1) of every output coordinate of a src -> dst resize."""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(np.float32)).astype(np.float32)
    if clamp:
        lo = s < 0
        f[lo], s[lo] = 0, 0
        hi = s >= src - 1
        f[hi], s[hi] = 0, src - 1
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return np.clip(s, 0, src - 1), np.clip(s + 1, 0, src - 1), a0, a1


def resize_u8(img, size):
    """cv2.resize(img, (size, size)) for a uint8 HxWxC image, INTER_LINEAR."""
    h, w, c = img.shape
    x0, x1, a0, a1 = coefficients(w, size, True)
    y0, y1, b0, b1 = coefficients(h, size, False)
    im = img.astype(np.int64)
    rows = im[:, x0] * a0[None, :, None] + im[:, x1] * a1[None, :, None]          # [h, size, c]
    h0, h1 = rows[y0], rows[y1]
    b0, b1 = b0[:, None, None], b1[:, None, None]
    out = ((((h0 >> 4) * b0) >> 16) + (((h1 >> 4) * b1) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def to_signed(u8):
    """The float step of utils/cv_utils.py:10-47 + models/imitator.py:89 on resized bytes: fp32 x / 255.0 * 2 - 1.0."""
    return u8.astype(np.float32) / 255.0 * 2 - 1.0


def kernel_float_steps(u8):
    """The kernel's float arithmetic, one fp32 rounding per step: __fdiv_rn, __fmul_rn, __fsub_rn."""
    x = np.asarray(u8).astype(np.float32)
    q = (x / np.float32(255)).astype(np.float32)
    return ((q * np.float32(2)).astype(np.float32) - np.float32(1)).astype(np.float32)


def frames(n, h, w, seed):
    """n random BGR uint8 frames [n,h,w,3], smooth enough to look like images and with every byte value present."""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
    ramp = (255 * (0.5 + 0.5 * np.sin(6 * xx + 4 * yy)))[None, :, :, None]
    mix = rng.random((n, 1, 1, 1)) < 0.5
    return np.where(mix, base, np.clip(ramp + rng.normal(0, 8, (n, h, w, 3)), 0, 255)).astype(np.uint8)


def cv2_route(frame, size, bgr=True, hmr_size=HMR_SIZE):
    """What the reference computes from one decoded frame with cv2 on the host (utils/cv_utils.py read_cv2_img,
    transform_img and save_cv2_img, the HMR resize of models/imitator.py:271-275), the result lwb_frames_in must
    reproduce: -> (img [3,S,S] fp32, hmr [3,224,224] fp32, gt_ image [S,S,3] uint8 BGR)."""
    import cv2
    rgb = cv2.cvtColor(frame, cv2.COLOR_BGR2RGB) if bgr else frame
    img = (cv2.resize(rgb, (size, size)).astype(np.float32) / 255.0).transpose((2, 0, 1)) * 2 - 1.0
    hmr = cv2.resize(rgb, (hmr_size, hmr_size)).astype(np.float32).transpose((2, 0, 1)) / 255.0 * 2 - 1.0
    gt = cv2.resize(cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR), (size, size))
    return img, hmr, gt
