"""The glue kernels around the conv engine against float64 restatements of their operations, at the shapes, channel
counts, pitches and value edges listed in glue_cases.py.  Every caller-allocated output is a view inside a sentinel
band that must come back unchanged; test_glue_cases_cpu.py runs the same cases through the CPU emulator."""
import pytest
import torch

from impersonator_b200 import kernels as K
import glue_cases as G
from conv_emulation import assert_bands_intact, guarded

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", G.CASES, ids=[c.name for c in G.CASES])
def test_glue_kernel(cuda, case):
    bufs = []

    def put(t):
        return None if t is None else t.to(cuda)

    def alloc(init):
        buf, view = guarded(cuda, tuple(init.shape), init.dtype, 0)
        view.copy_(init.to(cuda))
        bufs.append(buf)
        return view

    outs = case.run(K, put, alloc)
    torch.cuda.synchronize()
    for i, buf in enumerate(bufs):
        assert_bands_intact("%s buffer %d" % (case.name, i), buf)
    G.verify(case, {k: v.cpu() for k, v in outs.items()}, kernel=True)
