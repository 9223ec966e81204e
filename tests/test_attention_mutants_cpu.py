"""The strength of the self-attention bar (glue_cases.py): a float32 restatement of k_self_attention's algorithm -- 64-key
tiles, the running maximum and the per-key rescale of l and the accumulator, in the kernel's key order -- meets every
self_attention_nhwc case, and each mutant of it exceeds the bar at least 4x on at least one case.  CPU only.

Leaving out the key bias is not among the mutants: it shifts all logits of a query by the same q . bias_k, which the
softmax cancels, so no value check can see it.  Leaving out the query or the value bias can be seen, and is tested."""
import types

import pytest
import torch

import glue_cases as G

TILE = 64
CASES = [c for c in G.CASES if c.front == "self_attention_nhwc"]


def restated(mutant=None):
    """k_self_attention in float32, one 64-key tile at a time, the keys of a tile in order (cummax = the running
    maximum the kernel holds after each key).  mutant: None | drop_partial_tile | skip_acc_rescale | skip_l_rescale |
    no_query_bias | no_value_bias | swap_parts (the thread of part 0 reads the value slots of part 1 and vice versa)."""
    def self_attention_nhwc(qkv, bias, x, gamma, dq=G.ATT_DQ, out=None):
        n, h, w, _ = qkv.shape
        N, dv = h * w, x.shape[3]
        b = bias.clone()
        if mutant == "no_query_bias":
            b[:dq] = 0
        if mutant == "no_value_bias":
            b[2 * dq:] = 0
        t = (qkv[..., :2 * dq + dv] + b).view(n, N, -1)
        q, k, v = t[..., :dq], t[..., dq:2 * dq], t[..., 2 * dq:]
        if mutant == "swap_parts":      # float4 slot s of the value row belongs to part s % 4: swap parts 0 and 1
            slots = torch.arange(dv // 4).view(-1, 4)[:, [1, 0, 2, 3]].reshape(-1)
            v = v.view(n, N, dv // 4, 4)[:, :, slots].reshape(n, N, dv)
        m = torch.full((n, N, 1), float("-inf"))
        l = torch.zeros(n, N, 1)
        acc = torch.zeros(n, N, dv)
        for k0 in range(0, N, TILE):
            kn = min(TILE, N - k0)
            if mutant == "drop_partial_tile" and kn < TILE:
                break
            s = torch.bmm(q, k[:, k0:k0 + kn].transpose(1, 2))                    # [n, N, kn]
            run = torch.maximum(torch.cummax(s, dim=2).values, m)                 # the running max after each key
            m_end = run[..., -1:]
            p = torch.exp(s - run)                                                # each key's p against the max of its time
            late = torch.exp(run - m_end)                                         # the rescales that follow the key
            f0 = torch.exp(m - m_end)                                             # the tile's rescale of the old sums
            f0 = torch.where(torch.isinf(m), torch.zeros_like(f0), f0)
            l = (l if mutant == "skip_l_rescale" else l * f0) + (p if mutant == "skip_l_rescale" else p * late).sum(-1, keepdim=True)
            if mutant == "skip_acc_rescale":
                acc = acc + torch.bmm(p, v[:, k0:k0 + kn])
            else:
                acc = acc * f0 + torch.bmm(p * late, v[:, k0:k0 + kn])
            m = m_end
        y = (gamma * (acc * (1.0 / l)) + x.view(n, N, dv)).view(n, h, w, dv)
        out.copy_(y)
        return out
    return types.SimpleNamespace(self_attention_nhwc=self_attention_nhwc)


def _run(api, case):
    return case.run(api, lambda t: None if t is None else t.clone(), lambda init: init.clone())


def _worst(case, outs):
    """Largest err / bar over the case's Tol checks (0 for a case checked by Bits alone)."""
    r = 0.0
    for chk in case.checks:
        if isinstance(chk, G.Tol):
            ratio, _ = chk.ratio(case.name, outs)
            r = max(r, float(torch.nan_to_num(ratio, nan=float("inf")).max()))
    return r


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_restatement_meets_every_case(case):
    G.verify(case, _run(restated(), case), kernel=True)


MUTANTS = ["drop_partial_tile", "skip_acc_rescale", "skip_l_rescale", "no_query_bias", "no_value_bias", "swap_parts"]


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_exceeds_the_bar(mutant):
    api = restated(mutant)
    ratios = {c.edge: _worst(c, _run(api, c)) for c in CASES}
    for edge, r in sorted(ratios.items(), key=lambda kv: -kv[1]):
        print("%s / %s: err / bar %.3g" % (mutant, edge, r))
    best = max(ratios.values())
    print("%s: largest err / bar %.3g" % (mutant, best))
    assert best >= 4.0, "mutant %s stays within 4x the bar on every case (largest %.3g)" % (mutant, best)
