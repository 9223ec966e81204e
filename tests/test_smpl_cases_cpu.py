"""The strength of the smpl_forward bars (glue_cases.py): on the cases' random models, leaving out one beta, or a quarter
of the 207 pose terms, moves the float64 vertices by more than 10 bars.  CPU only."""
import pytest

import glue_cases as G
from oracle import smpl_ref

CASES = [c for c in G.CASES if c.front == "smpl_forward" and c.edge in ("batch=7", "num_betas=16", "V=6890", "wild poses")]


@pytest.mark.parametrize("drop", ["last beta", "a quarter of the pose terms"])
@pytest.mark.parametrize("case", CASES, ids=[c.edge for c in CASES])
def test_dropped_term_moves_vertices_past_10_bars(case, drop):
    m, beta, theta, rot, cam, refs = case.smpl
    m = dict(m)
    if drop == "last beta":
        m["shapedirs"] = m["shapedirs"].clone()
        m["shapedirs"][-1] = 0
    else:                                   # the pose bases of one K slice of the kernel's pose blend (k % 4 == 3)
        m["posedirs"] = m["posedirs"].clone()
        m["posedirs"][3::4] = 0
    verts = smpl_ref.forward(m, beta.double(), theta.double(), rotate_base=rot)[0]
    bar = G.SMPL_TAU * G.U32 * refs()["S"]["verts"]
    r = float(((verts - refs()["ref"]["verts"]).abs() / bar).max())
    print("%s, %s dropped: largest move %.1f bars" % (case.edge, drop, r))
    assert r > 10
