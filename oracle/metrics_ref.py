"""CPU restatement of his_evaluators' paired metrics (metrics/metrics.py:450-631), for the tests.

SSIM and PSNR restate skimage 0.16.2 as the metric classes call it, line by line, in float64 numpy with
scipy.ndimage.uniform_filter; LPIPS restates PNetLin(pnet_type='alex', version='0.1') (lpips/models/networks_basic.py
:65-168, pretrained_networks.py:58-96) in torch, with the weights as arguments.  Nothing here imports the reference.
"""
import numpy as np
import torch
import torch.nn.functional as F
from scipy.ndimage import uniform_filter

SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)
# (features index, stride, pad) of torchvision's alexnet().features convolutions; pools (3, 2) after conv1 and conv2
ALEX = ((0, 4, 2), (3, 1, 2), (6, 1, 1), (8, 1, 1), (10, 1, 1))


def preprocess(x):
    """metrics.py:456-476: [3,H,W] in [0,1] -> float32 HWC in [-1,1]."""
    out = np.asarray(x, dtype=np.float32).copy()
    out *= 2
    out -= 1
    return np.transpose(out, (1, 2, 0))


def structural_similarity(X, Y):
    """skimage.metrics.structural_similarity(X, Y, multichannel=True) (0.16.2) of two float32 HWC images."""
    nch = X.shape[-1]
    mssim = np.empty(nch)
    for ch in range(nch):
        mssim[ch] = _ssim_channel(X[..., ch], Y[..., ch], data_range=2.0)      # dtype_range[float32] = (-1, 1)
    return mssim.mean()


def _ssim_channel(X, Y, data_range, win_size=7, K1=0.01, K2=0.03):
    X = X.astype(np.float64)
    Y = Y.astype(np.float64)
    NP = win_size ** 2
    cov_norm = NP / (NP - 1)                                         # use_sample_covariance
    ux = uniform_filter(X, size=win_size)                            # mode 'reflect'
    uy = uniform_filter(Y, size=win_size)
    uxx = uniform_filter(X * X, size=win_size)
    uyy = uniform_filter(Y * Y, size=win_size)
    uxy = uniform_filter(X * Y, size=win_size)
    vx = cov_norm * (uxx - ux * ux)
    vy = cov_norm * (uyy - uy * uy)
    vxy = cov_norm * (uxy - ux * uy)
    R = data_range
    C1 = (K1 * R) ** 2
    C2 = (K2 * R) ** 2
    A1, A2, B1, B2 = (2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2)
    D = B1 * B2
    S = (A1 * A2) / D
    pad = (win_size - 1) // 2
    return S[pad:-pad, pad:-pad].mean()                               # crop(S, pad).mean()


def peak_signal_noise_ratio(image_true, image_test):
    """skimage.metrics.peak_signal_noise_ratio (0.16.2) of two float32 images, data_range from image_true."""
    dmin, dmax = -1.0, 1.0                                           # dtype_range[float32]
    true_min, true_max = np.min(image_true), np.max(image_true)
    if true_max > dmax or true_min < dmin:
        raise ValueError("im_true has intensity values outside the range expected for its data type")
    data_range = dmax if true_min >= 0 else dmax - dmin
    im1, im2 = np.asarray(image_true, np.float32), np.asarray(image_test, np.float32)
    err = np.mean((im1 - im2) ** 2, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return 10 * np.log10((data_range ** 2) / err)


def ssim_scores(preds, gts):
    """Per-frame SSIMMetric.forward of [N,3,H,W] frames in [0,1]."""
    return np.array([structural_similarity(preprocess(p), preprocess(g)) for p, g in zip(preds, gts)])


def psnr_scores(preds, gts):
    return np.array([peak_signal_noise_ratio(image_true=preprocess(g), image_test=preprocess(p)) for p, g in zip(preds, gts)])


def alexnet_features(x, convs):
    """relu1..relu5 of torchvision's alexnet().features (pretrained_networks.py:58-96); convs = [(w, b)] x 5."""
    outs = []
    h = x
    for k, ((w, b), (_, stride, pad)) in enumerate(zip(convs, ALEX)):
        if k in (1, 2):
            h = F.max_pool2d(h, 3, 2)
        h = F.relu(F.conv2d(h, w.to(h.dtype), b.to(h.dtype), stride=stride, padding=pad))
        outs.append(h)
    return outs


def normalize_tensor(x, eps=1e-10):
    """lpips/util/util.py:74-78."""
    return x / (torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True)) + eps)


def lpips(in0, in1, convs, lins, dtype=torch.float64):
    """PNetLin.forward(in0, in1) of [N,3,H,W] inputs in [-1,1] -> (val [N], per-layer values [N,5]).  PerceptualLoss
    calls it as forward_pair(target, pred): in0 = ref, in1 = pred.  lins = [lin_k of shape [c_k]]."""
    shift = torch.tensor(SHIFT, dtype=torch.float32).view(1, 3, 1, 1)
    scale = torch.tensor(SCALE, dtype=torch.float32).view(1, 3, 1, 1)
    # the scaling layer in the working dtype, with the float32 constants of networks_basic.py:102-103
    x0 = (in0.to(dtype) - shift.to(dtype)) / scale.to(dtype)
    x1 = (in1.to(dtype) - shift.to(dtype)) / scale.to(dtype)
    o0, o1 = alexnet_features(x0, convs), alexnet_features(x1, convs)
    layers = []
    for k in range(5):
        d = (normalize_tensor(o0[k]) - normalize_tensor(o1[k])) ** 2
        lin = lins[k].to(dtype).view(1, -1, 1, 1)
        layers.append(torch.mean(torch.mean(F.conv2d(d, lin), dim=3), dim=2)[:, 0])
    layers = torch.stack(layers, dim=1)
    val = layers[:, 0]
    for k in range(1, 5):
        val = val + layers[:, k]
    return val, layers


def perceptual_calculate_score(preds, gts, convs, lins, batch_size=32, dtype=torch.float64):
    """PerceptualMetric.calculate_score: the mean of per-chunk means of LPIPS(pred*2-1, gt*2-1)."""
    scores = []
    for i in range(int(np.ceil(len(preds) / batch_size))):
        p = torch.as_tensor(preds[i * batch_size:(i + 1) * batch_size]).float() * 2 - 1
        g = torch.as_tensor(gts[i * batch_size:(i + 1) * batch_size]).float() * 2 - 1
        scores.append(lpips(g, p, convs, lins, dtype)[0].mean())
    return torch.stack(scores).mean().item()
