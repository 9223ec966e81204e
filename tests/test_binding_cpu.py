"""Host wiring of the LPIPS and InceptionV3 streams on CPU against their oracles (kernel front-ends replaced by the torch
stand-ins of tests/kernel_emulator.py), and the weight packing every conv-engine stream shares."""
import os

import numpy as np
import torch

import inception_cases as IC
import kernel_emulator
import metrics_cases as MC
from impersonator_b200 import kernels as K, metrics as M, synthetic as S

CPU = torch.device("cpu")


def _cpu_metrics(monkeypatch):
    kernel_emulator.install(monkeypatch)
    monkeypatch.setattr(M, "_device", lambda device: CPU)
    torch.set_grad_enabled(False)


def test_lpips_stream_matches_oracle(monkeypatch):
    from oracle import metrics_ref as R
    _cpu_metrics(monkeypatch)
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    lp = M.LPIPS(weights=MC.alexnet_state_dict(convs), lin_weights=MC.lin_state_dict(lins))
    preds, gts = (torch.from_numpy(a) for a in MC.make_case("nonneg"))
    n, _, h, w = preds.shape
    score, layers = M._AlexStream(lp, n, h, w, CPU).run(preds, gts, True)
    ref, ref_layers = R.lpips(gts * 2 - 1, preds * 2 - 1, convs, lins)
    d = max((score.double() - ref).abs().max().item(), (layers.double() - ref_layers).abs().max().item())
    assert d < 1e-5 * ref.abs().max().item(), d


def test_inception_stream_matches_oracle(monkeypatch):
    from oracle import inception_ref as R
    _cpu_metrics(monkeypatch)
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inception.npz"))
    sd = IC.golden_state_dict(gold)
    frames = IC.make_case("wide")
    net = M.InceptionFeatures(weights=sd)
    f = net.stream(*frames.shape[:1], *frames.shape[2:]).run(torch.from_numpy(frames))
    ref = R.features(frames, sd)
    err = (f.double() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-5, err


def test_every_stream_packs_with_a_known_absmax(monkeypatch):
    """Each stream reads max|w| of all its layers in one host sync before packing: no pack call computes it itself."""
    from impersonator_b200.detectors import MaskRCNN, _DetStream
    from impersonator_b200.generator import ImpersonatorGenerator
    from impersonator_b200.hmr import HumanModelRecovery, _HmrStream
    from impersonator_b200.inpaintor import InpaintSANet, _InpaintStream
    _cpu_metrics(monkeypatch)
    calls = []

    def recorded(pack):
        def f(w, *args, **kw):
            calls.append(kw.get("absmax"))
            return pack(w, *args, **kw)
        return f
    monkeypatch.setattr(K, "pack_conv_weight", recorded(kernel_emulator.pack_conv_weight))
    monkeypatch.setattr(K, "pack_conv_weight_rowk", recorded(kernel_emulator.pack_conv_weight_rowk))
    gen = ImpersonatorGenerator(bg_dim=4, src_dim=6, tsf_dim=6, repeat_num=6).eval()
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inception.npz"))
    convs, lins = MC.synthetic_alexnet(), MC.synthetic_lins()
    builds = {
        "hmr": lambda: _HmrStream(HumanModelRecovery(smpl_model=S.synthetic_smpl_model(seed=3)).eval(), 1, CPU, 1),
        "inpaintor": lambda: _InpaintStream(InpaintSANet(c_dim=4).eval(), 1, 64, 64, CPU, 1),
        "detector": lambda: _DetStream(MaskRCNN(), 64, 64, CPU),
        "lpips": lambda: M._AlexStream(M.LPIPS(weights=MC.alexnet_state_dict(convs), lin_weights=MC.lin_state_dict(lins)),
                                       1, 64, 64, CPU),
        "inception": lambda: M.InceptionFeatures(weights=IC.golden_state_dict(gold)).stream(1, 64, 64),
        "unet": lambda: gen.tsf_model(torch.zeros(1, 6, 64, 64)),
        "bg": lambda: gen.bg_model(torch.zeros(1, 4, 64, 64)),
    }
    counts = {}
    for name, build in builds.items():
        del calls[:]
        build()
        assert calls and all(isinstance(a, float) for a in calls), (name, calls)
        counts[name] = len(calls)
    # the generator streams with the default (folded tensor-core) heads: stem, 3 encoders, 6 x 2 residual convs,
    # 3 decoders, 3 skippers (not in the BG net), heads
    assert counts == dict(hmr=52, inpaintor=36, detector=79, lpips=4, inception=65, unet=23, bg=20), counts
