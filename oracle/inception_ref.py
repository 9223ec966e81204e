"""CPU / GPU float64 restatement of his_evaluators' unpaired metrics (metrics/metrics.py:16-158, 309-395, 634-781), for
the tests.

``features`` restates InceptionV3(output_blocks=[3], resize_input=False, normalize_input=False) behind the metric
classes' preprocess (x * 2 - 1 in float32, bilinear resize to 299x299, align_corners=False) in torch without torchvision:
torchvision's Inception3 modules Conv2d_1a..Mixed_7c as conv (no bias) + eval-mode BatchNorm (eps 0.001) + ReLU, with
the state dict as argument.  ``frechet_distance`` and ``inception_score`` restate calculate_frechet_distance (scipy
sqrtm), fid_score_func and is_score_func in numpy.  Nothing here imports the reference or the product.
"""
import numpy as np
import torch
import torch.nn.functional as F
from scipy import linalg

EPS = 0.001


def preprocess(x, dtype=torch.float64, map_dtype=torch.float32):
    """metrics.py:645-669: [N,3,H,W] in [0,1] -> x * 2 - 1 (in ``map_dtype``: float32 for the float32 frames the metric
    classes get), bilinear to 299x299 in ``dtype``."""
    out = torch.as_tensor(x).to(map_dtype).clone()
    out *= 2
    out -= 1
    return F.interpolate(out.to(dtype), size=(299, 299), mode='bilinear', align_corners=False)


def _conv(x, sd, name, stride=1, padding=0):
    """torchvision BasicConv2d: relu(bn(conv(x))), eval-mode BatchNorm."""
    g = lambda k: sd[name + k].to(device=x.device, dtype=x.dtype)
    y = F.conv2d(x, g(".conv.weight"), None, stride=stride, padding=padding)
    y = F.batch_norm(y, g(".bn.running_mean"), g(".bn.running_var"), g(".bn.weight"), g(".bn.bias"), False, 0.0, EPS)
    return F.relu(y)


def _block_a(x, sd, b):
    b1 = _conv(x, sd, b + ".branch1x1")
    b5 = _conv(_conv(x, sd, b + ".branch5x5_1"), sd, b + ".branch5x5_2", padding=2)
    bd = _conv(_conv(_conv(x, sd, b + ".branch3x3dbl_1"), sd, b + ".branch3x3dbl_2", padding=1), sd,
               b + ".branch3x3dbl_3", padding=1)
    bp = _conv(F.avg_pool2d(x, 3, 1, 1), sd, b + ".branch_pool")
    return torch.cat([b1, b5, bd, bp], 1)


def _block_b(x, sd, b):
    b3 = _conv(x, sd, b + ".branch3x3", stride=2)
    bd = _conv(_conv(_conv(x, sd, b + ".branch3x3dbl_1"), sd, b + ".branch3x3dbl_2", padding=1), sd,
               b + ".branch3x3dbl_3", stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, 3, 2)], 1)


def _block_c(x, sd, b):
    b1 = _conv(x, sd, b + ".branch1x1")
    b7 = _conv(x, sd, b + ".branch7x7_1")
    b7 = _conv(b7, sd, b + ".branch7x7_2", padding=(0, 3))
    b7 = _conv(b7, sd, b + ".branch7x7_3", padding=(3, 0))
    bd = _conv(x, sd, b + ".branch7x7dbl_1")
    for k, p in ((2, (3, 0)), (3, (0, 3)), (4, (3, 0)), (5, (0, 3))):
        bd = _conv(bd, sd, b + ".branch7x7dbl_%d" % k, padding=p)
    bp = _conv(F.avg_pool2d(x, 3, 1, 1), sd, b + ".branch_pool")
    return torch.cat([b1, b7, bd, bp], 1)


def _block_d(x, sd, b):
    b3 = _conv(_conv(x, sd, b + ".branch3x3_1"), sd, b + ".branch3x3_2", stride=2)
    b7 = _conv(x, sd, b + ".branch7x7x3_1")
    b7 = _conv(b7, sd, b + ".branch7x7x3_2", padding=(0, 3))
    b7 = _conv(b7, sd, b + ".branch7x7x3_3", padding=(3, 0))
    b7 = _conv(b7, sd, b + ".branch7x7x3_4", stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, 3, 2)], 1)


def _block_e(x, sd, b):
    b1 = _conv(x, sd, b + ".branch1x1")
    b3 = _conv(x, sd, b + ".branch3x3_1")
    b3 = torch.cat([_conv(b3, sd, b + ".branch3x3_2a", padding=(0, 1)), _conv(b3, sd, b + ".branch3x3_2b", padding=(1, 0))], 1)
    bd = _conv(_conv(x, sd, b + ".branch3x3dbl_1"), sd, b + ".branch3x3dbl_2", padding=1)
    bd = torch.cat([_conv(bd, sd, b + ".branch3x3dbl_3a", padding=(0, 1)), _conv(bd, sd, b + ".branch3x3dbl_3b", padding=(1, 0))], 1)
    bp = _conv(F.avg_pool2d(x, 3, 1, 1), sd, b + ".branch_pool")
    return torch.cat([b1, b3, bd, bp], 1)


def network(x, sd, taps=None):
    """Blocks 0..3 of InceptionV3 on a preprocessed [N,3,299,299] batch -> [N,2048].  ``taps``: a dict that receives
    NCHW activations after 'stem' (Conv2d_1a), 'mixed_5d', 'mixed_6e' and 'mixed_7c'."""
    taps = {} if taps is None else taps
    x = _conv(x, sd, "Conv2d_1a_3x3", stride=2)
    taps["stem"] = x
    x = _conv(x, sd, "Conv2d_2a_3x3")
    x = F.max_pool2d(_conv(x, sd, "Conv2d_2b_3x3", padding=1), 3, 2)
    x = F.max_pool2d(_conv(_conv(x, sd, "Conv2d_3b_1x1"), sd, "Conv2d_4a_3x3"), 3, 2)
    for b in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        x = _block_a(x, sd, b)
    taps["mixed_5d"] = x
    x = _block_b(x, sd, "Mixed_6a")
    for b in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        x = _block_c(x, sd, b)
    taps["mixed_6e"] = x
    x = _block_d(x, sd, "Mixed_7a")
    x = _block_e(x, sd, "Mixed_7b")
    x = _block_e(x, sd, "Mixed_7c")
    taps["mixed_7c"] = x
    return F.adaptive_avg_pool2d(x, 1)[:, :, 0, 0]


def features(frames, sd, device="cpu", taps=None, map_dtype=torch.float32):
    """FIDMetric.forward in float64: [N,3,H,W] frames in [0,1] -> [N,2048]."""
    with torch.no_grad():
        return network(preprocess(frames, map_dtype=map_dtype).to(device), sd, taps)


def frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """calculate_frechet_distance (metrics.py:309-361) with scipy's sqrtm."""
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    diff = mu1 - mu2
    covmean = linalg.sqrtm(sigma1.dot(sigma2))
    if not np.isfinite(covmean).all():
        offset = np.eye(sigma1.shape[0]) * eps
        covmean = linalg.sqrtm((sigma1 + offset).dot(sigma2 + offset))
    if np.iscomplexobj(covmean):
        if not np.allclose(np.diagonal(covmean).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(covmean.imag))))
        covmean = covmean.real
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(covmean)


def frechet_distance_eig(mu1, sigma1, mu2, sigma2):
    """The same distance with tr sqrtm(s1 s2) = sum sqrt(max(l, 0)) over the eigenvalues l of the symmetric
    s1^1/2 s2 s1^1/2 (numpy eigh): real also where scipy's sqrtm of a rank-deficient product has imaginary parts."""
    lam, v = np.linalg.eigh(sigma1)
    r1 = (v * np.sqrt(np.maximum(lam, 0))) @ v.T
    m = r1 @ sigma2 @ r1
    tr = np.sqrt(np.maximum(np.linalg.eigvalsh((m + m.T) / 2), 0)).sum()
    diff = mu1 - mu2
    return diff.dot(diff) + np.trace(sigma1) + np.trace(sigma2) - 2 * tr


def fid_eig(pred_feats, gt_feats):
    return frechet_distance_eig(np.mean(pred_feats, axis=0), np.cov(pred_feats, rowvar=False),
                                np.mean(gt_feats, axis=0), np.cov(gt_feats, rowvar=False))


def fid(pred_feats, gt_feats):
    """fid_score_func (metrics.py:363-379)."""
    if len(pred_feats) == 0 or len(gt_feats) == 0:
        return 0
    return frechet_distance(np.mean(pred_feats, axis=0), np.cov(pred_feats, rowvar=False),
                            np.mean(gt_feats, axis=0), np.cov(gt_feats, rowvar=False))


def inception_score(feats_softmax):
    """is_score_func (metrics.py:381-395)."""
    kl = feats_softmax * (np.log(feats_softmax) - np.log(np.expand_dims(np.mean(feats_softmax, 0), 0)))
    return np.exp(np.mean(np.sum(kl, 1)))


def softmax64(feats):
    """F.softmax(feats, dim=1) in float64 numpy."""
    f = np.asarray(feats, dtype=np.float64)
    e = np.exp(f - f.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)
