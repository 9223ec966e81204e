"""Unit parity of the inpaintor glue kernels (lwb_gated_act_nhwc, lwb_self_attention_nhwc) against plain torch fp32."""
import pytest
import torch
import torch.nn.functional as F

from impersonator_b200 import kernels as K

pytestmark = pytest.mark.gpu


def test_self_attention_matches_torch(cuda):
    g = torch.Generator().manual_seed(0)
    n, h, w = 2, 24, 20                                   # 480 positions: not a multiple of the 64-wide tiles
    qkv = torch.randn(n, h, w, 160, generator=g)
    bias = torch.randn(160, generator=g) * 0.1
    x = torch.randn(n, h, w, 128, generator=g)
    gamma = torch.tensor([0.7])
    out = K.self_attention_nhwc(qkv.to(cuda), bias.to(cuda), x.to(cuda), gamma.to(cuda)).cpu()
    t = (qkv + bias).view(n, h * w, 160)
    q, k, v = t[..., :16], t[..., 16:32], t[..., 32:]
    att = torch.softmax(torch.bmm(q, k.transpose(1, 2)), dim=-1)                  # networks/inpaintor.py:97-99
    ref = (gamma * torch.bmm(att, v) + x.view(n, h * w, 128)).view(n, h, w, 128)   # :101-104 in NHWC
    d = (out - ref).abs().max().item()
    print("self attention vs torch: %.3e" % d)
    assert d < 2e-5


@pytest.mark.parametrize("c,c_stride,up,lo_format", [(16, 32, 1, 0), (3, 16, 1, 0), (64, 128, 2, 1), (32, 64, 2, 0)])
def test_gated_epilogue_matches_torch(cuda, c, c_stride, up, lo_format):
    g = torch.Generator().manual_seed(c)
    n, h, w = 2, 12, 10
    raw = torch.randn(n, h, w, c_stride, generator=g)
    bias = torch.randn(2 * c, generator=g) * 0.2
    scale = 1 + 0.2 * torch.randn(c, generator=g)
    shift = 0.1 * torch.randn(c, generator=g)
    a, b = raw[..., :c] + bias[:c], raw[..., c:2 * c] + bias[c:]
    ref = (F.leaky_relu(a, 0.2) * torch.sigmoid(b)) * scale + shift                # networks/inpaintor.py:37-47
    ref = ref.clamp(-1, 1)
    ref = ref.repeat_interleave(up, dim=1).repeat_interleave(up, dim=2)            # nearest 2x (:67)
    c_pad = 64
    y = torch.full((n, h * up, w * up, c), float("nan"), device=cuda)
    hi = torch.full((n, h * up, w * up, c_pad), float("nan"), dtype=torch.float16, device=cuda)
    lo = torch.empty_like(hi)
    K.gated_act_nhwc(raw.to(cuda), c, bias.to(cuda), 2, scale.to(cuda), shift.to(cuda), upsample=up, clamp=True,
                     y_f32=y, y_hi=hi, y_lo=lo, lo_format=lo_format)
    assert (y.cpu() - ref).abs().max().item() < 1e-5
    assert (hi[..., :c].float().cpu() - ref).abs().max().item() < 1e-3
    if c < c_pad:
        assert float(hi[..., c:].float().abs().max()) == 0.0                       # zero-padded K channels
    if lo_format == 0:
        assert ((hi.float() + lo.float())[..., :c].cpu() - ref).abs().max().item() < 1e-5


def _attention_args(cuda, n=1, h=3, w=5, dv=128):
    return (torch.zeros(n, h, w, 160, device=cuda), torch.zeros(160, device=cuda), torch.zeros(n, h, w, dv, device=cuda),
            torch.ones(1, device=cuda))


@pytest.mark.parametrize("bad", ["x batch", "x grid", "bias length", "out shape"])
def test_self_attention_rejects_mismatched_shapes(cuda, bad):
    qkv, bias, x, gamma = _attention_args(cuda)
    out = None
    if bad == "x batch":
        x = torch.zeros(2, 3, 5, 128, device=cuda)
    elif bad == "x grid":
        x = torch.zeros(1, 5, 3, 128, device=cuda)
    elif bad == "bias length":
        bias = torch.zeros(144, device=cuda)
    else:
        out = torch.zeros(1, 3, 4, 128, device=cuda)
    with pytest.raises(K.LwbError):
        K.self_attention_nhwc(qkv, bias, x, gamma, out=out)


def test_gated_act_rejects_lo_of_another_shape(cuda):
    raw = torch.zeros(1, 3, 5, 32, device=cuda)
    hi = torch.zeros(1, 3, 5, 64, dtype=torch.float16, device=cuda)
    lo = torch.zeros(1, 3, 4, 64, dtype=torch.float16, device=cuda)
    with pytest.raises(K.LwbError):
        K.gated_act_nhwc(raw, 16, None, 2, None, None, y_hi=hi, y_lo=lo)
