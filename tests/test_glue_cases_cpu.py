"""The glue cases of glue_cases.py through kernel_emulator's stand-ins, with the checks the GPU kernels meet: the host
orchestration the CPU suite validates on the emulator then rests on the same contract as the kernels.  Also checks that
every front-end the emulator replaces has its cases here or names the test that covers its kernel."""
import ast
import os

import pytest

import glue_cases as G
import kernel_emulator as E

HERE = os.path.dirname(os.path.abspath(__file__))
EMULATED = [c for c in G.CASES if c.emulated]


@pytest.mark.parametrize("case", EMULATED, ids=[c.name for c in EMULATED])
def test_emulator_meets_the_kernel_contract(case):
    outs = case.run(E, lambda t: None if t is None else t.clone(), lambda init: init.clone())
    G.verify(case, outs, kernel=False)


class _Recorder(object):
    def __init__(self):
        self.names = []

    def setattr(self, target, name, value):
        self.names.append(name)

    def setenv(self, name, value):
        pass


def _patched_names():
    rec = _Recorder()
    E.install_tasks(rec)
    return rec.names


def _test_functions(fname):
    with open(os.path.join(HERE, fname)) as f:
        tree = ast.parse(f.read())
    return {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}


def test_every_emulated_front_end_is_covered():
    covered = {}
    for c in G.CASES:
        covered.setdefault(c.front, []).append(c.edge)
    problems = []
    for name in sorted(set(_patched_names()) | set(G.REQUIRED_EDGES)):
        if name in G.COVERED_ELSEWHERE:
            fname, fn = G.COVERED_ELSEWHERE[name].split("::")
            if not os.path.exists(os.path.join(HERE, fname)) or fn not in _test_functions(fname):
                problems.append("%s: COVERED_ELSEWHERE names %s, which does not exist" % (name, G.COVERED_ELSEWHERE[name]))
            continue
        if name not in G.REQUIRED_EDGES:
            problems.append("%s: no glue case and no COVERED_ELSEWHERE entry" % name)
            continue
        missing = [e for e in G.REQUIRED_EDGES[name] if e not in covered.get(name, [])]
        if missing:
            problems.append("%s: no case for %s" % (name, ", ".join(missing)))
    assert not problems, "\n".join(problems)


def test_every_inpaintor_gated_binding_has_a_case(monkeypatch):
    """The (c, c_stride, up, outputs, lo_format) of every gated epilogue the inpaintor binds at 256x256, in all three
    precision modes, is one of the gated_act_nhwc cases."""
    E.install(monkeypatch)
    bound = G.inpaintor_gated_bindings()
    print("\n".join(str(b) for b in bound))
    assert bound == sorted(G.INPAINTOR_GATED)


def test_cases_are_the_required_edges():
    names = [c.name for c in G.CASES]
    assert len(names) == len(set(names)), "duplicate case names"
    extra = [c.name for c in G.CASES if c.edge not in G.REQUIRED_EDGES.get(c.front, [])]
    assert not extra, "cases outside REQUIRED_EDGES: %s" % extra
