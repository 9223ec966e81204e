"""The strength of the correspondence checks (correspond_cases.py): kernel_emulator.correspond meets every emulated
``correspond`` case (test_glue_cases_cpu.py), and the same stand-in with exactly one deliberate change exceeds some case's
bar at least 4x, or breaks one of its exact (Bits) contracts.  CPU only."""
import types

import pytest
import torch

import glue_cases as G
import kernel_emulator as E

CASES = [c for c in G.CASES if c.front == "correspond" and c.emulated]


def mutated(mutant):
    """kernel_emulator.correspond with one change: align_corners flipped | T's barycentric weights rotated by one vertex
    (T = sum_k w_k p2v[k - 1]) | the background cond row taken as row 0 | frame 0's source used for every frame |
    the vertical flip of every map dropped."""
    def correspond(cam, verts, face_idx, image_size, map_fn, src_p2verts, src_img=None, align_corners=None, out=None, **kw):
        if mutant == "align_corners flipped":
            align_corners = not align_corners
        elif mutant == "T weights rotated":
            src_p2verts = src_p2verts.roll(1, dims=2)
        elif mutant == "background cond row 0":
            map_fn = map_fn.clone()
            map_fn[-1] = map_fn[0]
        elif mutant == "frame 0 source":
            src_p2verts = src_p2verts[:1]
            src_img = src_img[:1] if src_img is not None else None
        res = E.correspond(cam, verts, face_idx, image_size, map_fn, src_p2verts, src_img, align_corners=align_corners,
                           out=out, **kw)
        if mutant == "no vertical flip":
            for k, dim in (("fim", 1), ("wim", 1), ("T", 1), ("tsf_inputs", 2)):
                res[k].copy_(res[k].flip(dim))
        return res
    return types.SimpleNamespace(correspond=correspond)


def _worst(case, outs):
    """Largest err / bar over the case's Tol checks; inf when one of its Bits checks fails."""
    r = 0.0
    for chk in case.checks:
        if isinstance(chk, G.Tol):
            ratio, _ = chk.ratio(case.name, outs)
            r = max(r, float(torch.nan_to_num(ratio, nan=float("inf")).max()) if ratio.numel() else 0.0)
        else:
            try:
                chk(case.name, outs)
            except AssertionError:
                r = float("inf")
    return r


MUTANTS = ["align_corners flipped", "T weights rotated", "background cond row 0", "frame 0 source", "no vertical flip"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_exceeds_the_bar(mutant):
    api = mutated(mutant)
    ratios = {c.edge: _worst(c, c.run(api, lambda t: None if t is None else t.clone(), lambda init: init.clone()))
              for c in CASES}
    for edge, r in sorted(ratios.items(), key=lambda kv: -kv[1]):
        print("%s / %s: err / bar %.3g" % (mutant, edge, r))
    best = max(ratios.values())
    print("%s: largest err / bar %.3g" % (mutant, best))
    assert best >= 4.0, "mutant %s stays within 4x the bar on every case (largest %.3g)" % (mutant, best)
