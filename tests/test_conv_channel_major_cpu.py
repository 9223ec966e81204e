"""CPU models of the channel-major conv tiles (conv_tc.cu): where each accumulator register of a consumer thread lands
in the output and the statistics, and the ring protocol between the producer and two consumer warpgroups that never
wait for each other.

1. Fragment mapping.  The value of GEMM element (image, pixel, N column) is a random table.  Each consumer warpgroup's
   wgmma result is read through the operand rows its descriptors address (weight rows from the B-ring entry offset,
   pixels from the activation box offset), split into the per-thread accumulator fragment of an M64 x N wgmma, and
   scattered with the epilogue's address arithmetic.  Pixel-major N = 16 / 32 tiles and channel-major N = 64 / 128 tiles
   must both reproduce the table at its NHWC offsets, merged transposed plans included, with partial tiles at the domain
   edges, and every thread's quad-reduced channel sums must add up to the per-image statistics.
2. Ring protocol.  The producer and the 8 consumer warps run the loops of k_conv_wg over each generator plan's geometry
   as coroutines on mbarriers with phase parity, one warpgroup delayed by random amounts: no entry is refilled before all
   8 warps released it, no warp reads an entry before it holds that warp's (tile, group, chunk, tap), nothing deadlocks.
"""
import importlib.util
import os
import random

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("conv_microbench", os.path.join(ROOT, "tools", "conv_microbench.py"))
MB = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MB)

TILE_H, TILE_W, ROW_BYTES, KCHUNK = 16, 8, 1024, 64
RING_BYTES, MAX_STAGES = 200 * 1024, 8


def tile_rows(n_tile):
    return 32 if n_tile == 64 else TILE_H


# ----------------------------------------------------------------------------------------------- fragment mapping
def fragment(n):
    """Accumulator fragment of an M64 x N wgmma: (row, column) of d[4j + 2h + e] for each of the 128 threads of a
    warpgroup, as [128, n / 2] arrays."""
    t = np.arange(128)[:, None]
    i = np.arange(n // 2)[None, :]
    w, lane = t // 32, t % 32
    j, h, e = i // 4, (i // 2) % 2, i % 2
    return 16 * w + lane // 4 + 8 * h, 8 * j + 2 * (lane % 4) + e


def run_epilogues(geo, V):
    """Every tile of the plan through the kernel's operand addressing, fragment and epilogue; returns (out, stats)."""
    n_tile, ncols, cout, pc = geo["n_tile"], geo["ncols"], geo["cout"], geo["phase_cols"]
    n_img, dom_h, dom_w = V.shape[:3]
    th = tile_rows(n_tile)
    out_h, out_w = geo["oy_mul"] * dom_h, geo["ox_mul"] * dom_w
    out = np.full(n_img * out_h * out_w * cout, np.nan)
    hits = np.zeros(out.size, int)
    stats = np.zeros((n_img, cout, 2))
    cm = n_tile >= 64
    for img in range(n_img):
        for ty in range(-(-dom_h // th)):
            for tx in range(-(-dom_w // TILE_W)):
                for n_idx in range(ncols // n_tile):
                    y0, x0 = ty * th, tx * TILE_W
                    for wg in range(2):
                        if cm:
                            # A = weight rows from b_base + wg * 64 * 128 (N = 128), B = 128 pixels from box row
                            # a_base / 1024 (N = 64: 16 wg); D^T[channel, pixel]
                            ch_off = 64 * wg if n_tile == 128 else 0
                            row_off = 0 if n_tile == 128 else 16 * wg
                            r, c = fragment(128)
                            chan, py, px = ch_off + r, row_off + c // 8, c % 8
                        else:
                            # A = 64 pixels from box row 8 wg, B = all n_tile weight rows; D[pixel, channel]
                            r, c = fragment(n_tile)
                            chan, py, px = c, 8 * wg + r // 8, r % 8
                        val = np.zeros(chan.shape)
                        inside = (y0 + py < dom_h) & (x0 + px < dom_w)
                        val[inside] = V[img, (y0 + py)[inside], (x0 + px)[inside], (n_idx * n_tile + chan)[inside]]
                        if cm:
                            epilogue_channel_major(geo, val, img, y0, x0, n_idx, wg, out_h, out_w, out, hits, stats)
                        else:
                            epilogue_plain(geo, val, img, y0, x0, n_idx, wg, out_h, out_w, out, hits, stats)
    assert hits.max() <= 1, "an output element is written twice"
    return out.reshape(n_img, out_h, out_w, cout), stats, hits


def epilogue_channel_major(geo, acc, img, y0t, x0t, n_idx, wg, out_h, out_w, out, hits, stats):
    """epilogue_channel_major of conv_tc.cu, for all 128 threads of warpgroup wg at once."""
    n_tile, cout, pc = geo["n_tile"], geo["cout"], geo["phase_cols"]
    dom_h, dom_w = geo["dom"]
    t = np.arange(128)
    warp, lane = 4 * wg + t // 32, t % 32
    c_base, row0 = (64 * wg, 0) if n_tile == 128 else (0, 16 * wg)
    y0, x0 = y0t + row0, x0t + 2 * (lane % 4)
    rows = dom_h - y0
    ch, coff = [], []
    for h in range(2):
        col = n_idx * n_tile + c_base + 16 * (warp % 4) + lane // 4 + 8 * h
        ph = col // pc if pc > 0 else np.zeros_like(col)
        ch.append(col - ph * pc)
        coff.append(((ph >> 1) * out_w + (ph & 1)) * cout + ch[-1])
    s, q = np.zeros((2, 128)), np.zeros((2, 128))
    for j in range(16):
        orow = (img * out_h + (geo["oy_mul"] * (y0 + j) + geo["oy_add"])) * out_w
        for e in range(2):
            v = (j < rows) & (x0 + e < dom_w)
            base = (orow + (geo["ox_mul"] * (x0 + e) + geo["ox_add"])) * cout
            for h in range(2):
                a = acc[:, 4 * j + 2 * h + e]
                o = (base + coff[h])[v]
                out[o] = a[v]
                hits[o] += 1
                s[h] += np.where(v, a, 0.0)
                q[h] += np.where(v, a * a, 0.0)
    for h in range(2):                                   # two quad shuffles, then the quad leader's atomics
        s_q, q_q = s[h].reshape(32, 4).sum(1), q[h].reshape(32, 4).sum(1)
        leaders = ch[h][::4]
        np.add.at(stats[img, :, 0], leaders, s_q)
        np.add.at(stats[img, :, 1], leaders, q_q)


def epilogue_plain(geo, acc, img, y0t, x0t, n_idx, wg, out_h, out_w, out, hits, stats):
    """epilogue_plain of conv_tc.cu (pixel-major), for all 128 threads of warpgroup wg at once."""
    n_tile, cout, pc = geo["n_tile"], geo["cout"], geo["phase_cols"]
    dom_h, dom_w = geo["dom"]
    t = np.arange(128)
    warp, lane = 4 * wg + t // 32, t % 32
    x = x0t + lane // 4
    for h in range(2):
        y = y0t + 2 * warp + h
        v = (y < dom_h) & (x < dom_w)
        for j in range(n_tile // 8):
            for e in range(2):
                c = 8 * j + 2 * (lane % 4) + e
                col = n_idx * n_tile + c
                ph = col // pc if pc > 0 else np.zeros_like(col)
                o = ((img * out_h + geo["oy_mul"] * y + geo["oy_add"] + (ph >> 1)) * out_w
                     + geo["ox_mul"] * x + geo["ox_add"] + (ph & 1)) * cout + col - ph * pc
                a = acc[:, 4 * j + 2 * h + e]
                out[o[v]] = a[v]
                hits[o[v]] += 1
                np.add.at(stats[img, :, 0], (col - ph * pc)[v], a[v])
                np.add.at(stats[img, :, 1], (col - ph * pc)[v], a[v] ** 2)


def reference(geo, V):
    """NHWC output and per-(image, channel) sums of the GEMM table, straight from the plan's definition."""
    n_img, dom_h, dom_w, ncols = V.shape
    cout, pc = geo["cout"], geo["phase_cols"]
    out = np.full((n_img, geo["oy_mul"] * dom_h, geo["ox_mul"] * dom_w, cout), np.nan)
    if pc:
        for ph in range(4):
            out[:, ph >> 1::2, ph & 1::2, :] = V[..., ph * pc:(ph + 1) * pc]
        vals = V.reshape(n_img, dom_h * dom_w * 4, cout)
    else:
        out[:, geo["oy_add"]::geo["oy_mul"], geo["ox_add"]::geo["ox_mul"], :] = V
        vals = V.reshape(n_img, dom_h * dom_w, cout)
    return out, np.stack([vals.sum(1), (vals ** 2).sum(1)], -1)


GEOMETRIES = {
    # plain stride-1 / stride-2 layers: cout 256 as two N tiles of 128, edge tiles in both directions
    "n128": dict(n_tile=128, cout=256, dom=(37, 13)),
    "n128_small": dict(n_tile=128, cout=128, dom=(5, 3)),
    # 4-phase transposed conv: one launch per phase writes every second output pixel
    "n128_phase": dict(n_tile=128, cout=128, dom=(19, 11), oy_mul=2, ox_mul=2, oy_add=1, ox_add=0),
    # merged transposed convs: the N columns are the four sub-pixel phases of cout channels
    "merged_cout64": dict(n_tile=128, cout=64, dom=(21, 10), merged=True),
    "merged_cout32": dict(n_tile=128, cout=32, dom=(9, 17), merged=True),
    "merged_cout128": dict(n_tile=128, cout=128, dom=(17, 9), merged=True),
    # channel-major 256-pixel tiles (stem, 64+64 -> 64 skipper)
    "n64": dict(n_tile=64, cout=64, dom=(45, 20)),
    "n64_two": dict(n_tile=64, cout=192, dom=(33, 7)),
    # pixel-major folded heads
    "n32": dict(n_tile=32, cout=64, dom=(19, 9)),
    "n16": dict(n_tile=16, cout=16, dom=(17, 15)),
}


def _geo(name):
    g = dict(GEOMETRIES[name])
    g.setdefault("oy_mul", 1), g.setdefault("ox_mul", 1), g.setdefault("oy_add", 0), g.setdefault("ox_add", 0)
    if g.pop("merged", False):
        g.update(oy_mul=2, ox_mul=2, phase_cols=g["cout"], ncols=4 * g["cout"])
    else:
        g.update(phase_cols=0, ncols=g["cout"])
    return g


@pytest.mark.parametrize("name", sorted(GEOMETRIES))
def test_fragment_mapping_reproduces_the_gemm(name):
    geo = _geo(name)
    rng = np.random.default_rng(7)
    V = rng.standard_normal((2, geo["dom"][0], geo["dom"][1], geo["ncols"]))
    out, stats, hits = run_epilogues(geo, V)
    ref_out, ref_stats = reference(geo, V)
    np.testing.assert_array_equal(np.isnan(out), np.isnan(ref_out))
    np.testing.assert_array_equal(out[~np.isnan(ref_out)], ref_out[~np.isnan(ref_out)])
    assert hits.sum() == V.size
    np.testing.assert_allclose(stats, ref_stats, rtol=1e-12, atol=1e-12)


def test_channel_major_matches_pixel_major_at_n128():
    """The same N = 128 plan through the parent's pixel-major fragment and the channel-major one."""
    geo = _geo("merged_cout64")
    V = np.random.default_rng(3).standard_normal((2, geo["dom"][0], geo["dom"][1], geo["ncols"]))
    cm, cm_stats, _ = run_epilogues(geo, V)
    geo_pm = dict(geo, n_tile=32)          # pixel-major fragment, same 16 x 8 tiles, four N tiles per 128 columns
    pm, pm_stats, _ = run_epilogues(geo_pm, V)
    np.testing.assert_array_equal(cm, pm)
    np.testing.assert_allclose(cm_stats, pm_stats, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------- ring protocol
class MBarrier:
    """mbarrier with an arrival count per phase; wait(parity) passes once the phase of that parity has completed."""

    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def ready(self, parity):
        return (self.phase & 1) != parity


def plan_geometry(spec, n_tile, split):
    """(taps per group, chunks, A stages, B stages) of each launch of a plan: group_taps + pick_rings of conv_tc.cu."""
    chunks = 1 if spec["kind"] == "rowk" else (spec["cin"] + spec.get("cin1", 0)) // KCHUNK
    ops = 2 if split else 1
    out = []
    for taps in MB.launch_taps(spec):
        cnts, prev = [], None
        for v, dy, dx in sorted(taps, key=lambda t: (t[0], t[2], t[1])):
            if prev is not None and (v, dx) == (prev[0], prev[2]) and dy == prev[1] + 1 and cnts[-1] < 8:
                cnts[-1] += 1
            else:
                cnts.append(1)
            prev = (v, dy, dx)
        a_rows = tile_rows(n_tile) + max(cnts) - 1
        a_bytes, b_bytes = a_rows * ROW_BYTES * ops, n_tile * 128 * ops
        best, stages = 0, None
        for a in range(2, MAX_STAGES + 1):
            b = min(MAX_STAGES, (RING_BYTES - a * a_bytes) // b_bytes)
            if b < 2:
                break
            if min(a * max(cnts), b) > best:
                best, stages = min(a * max(cnts), b), (a, b)
        out.append((cnts, chunks, stages[0], stages[1]))
    return out


def simulate(cnts, chunks, a_stages, b_stages, tiles, seed, slow_wg):
    """Runs the producer and the 8 consumer warps of one CTA over `tiles` tiles; warpgroup slow_wg stalls at random."""
    rng = random.Random(seed)
    a_full = [MBarrier(1) for _ in range(a_stages)]
    a_empty = [MBarrier(8) for _ in range(a_stages)]
    b_full = [MBarrier(1) for _ in range(b_stages)]
    b_empty = [MBarrier(8) for _ in range(b_stages)]
    a_tag, b_tag = [None] * a_stages, [None] * b_stages         # what an entry holds
    a_rel, b_rel = [set(range(8)) for _ in range(a_stages)], [set(range(8)) for _ in range(b_stages)]

    def producer():
        as_ = bs = 0
        aph = bph = 0
        for tile in range(tiles):
            for g, cnt in enumerate(cnts):
                for chunk in range(chunks):
                    yield lambda s=as_, p=aph ^ 1: a_empty[s].ready(p)
                    assert a_rel[as_] == set(range(8)), "A entry refilled before every consumer warp released it"
                    a_tag[as_], a_rel[as_] = (tile, g, chunk), set()
                    a_full[as_].arrive()                          # TMA completion
                    as_ += 1
                    if as_ == a_stages:
                        as_, aph = 0, aph ^ 1
                    for i in range(cnt):
                        yield lambda s=bs, p=bph ^ 1: b_empty[s].ready(p)
                        assert b_rel[bs] == set(range(8)), "B entry refilled before every consumer warp released it"
                        b_tag[bs], b_rel[bs] = (tile, g, chunk, i), set()
                        b_full[bs].arrive()
                        bs += 1
                        if bs == b_stages:
                            bs, bph = 0, bph ^ 1

    def release(warp, a, b):
        if b is not None:
            assert warp not in b_rel[b]
            b_rel[b].add(warp)
            b_empty[b].arrive()
        if a is not None:
            assert warp not in a_rel[a]
            a_rel[a].add(warp)
            a_empty[a].arrive()

    def consumer(warp):
        as_ = bs = 0
        aph = bph = 0
        for tile in range(tiles):
            prev_b = prev_a = None
            for g, cnt in enumerate(cnts):
                for chunk in range(chunks):
                    yield lambda s=as_, p=aph: a_full[s].ready(p)
                    for i in range(cnt):
                        yield lambda s=bs, p=bph: b_full[s].ready(p)
                        # the wgmma group reads both entries
                        assert a_tag[as_] == (tile, g, chunk), "A entry read before it holds this chunk"
                        assert b_tag[bs] == (tile, g, chunk, i), "B entry read before it holds this tap"
                        if prev_b is not None:                  # wgmma.wait_group 1: the previous group retired
                            release(warp, prev_a, prev_b)
                            prev_a = None
                        prev_b = bs
                        bs += 1
                        if bs == b_stages:
                            bs, bph = 0, bph ^ 1
                    prev_a = as_
                    as_ += 1
                    if as_ == a_stages:
                        as_, aph = 0, aph ^ 1
            release(warp, prev_a, prev_b)                      # wgmma.wait_group 0, then the epilogue: no barrier
            for _ in range(rng.randrange(4)):
                yield lambda: True

    agents = [producer()] + [consumer(w) for w in range(8)]
    waits = [None] * len(agents)
    live = set(range(len(agents)))
    slow = lambda k: 1 <= k <= 8 and (k - 1) // 4 == slow_wg    # noqa: E731
    delay = rng.choice((0.5, 0.9, 0.99))
    while live:
        runnable = [k for k in live if waits[k] is None or waits[k]()]
        if not runnable:
            raise AssertionError("deadlock: no agent can proceed")
        k = rng.choice(runnable)
        if slow(k) and rng.random() < delay and not all(slow(o) for o in runnable):
            continue                                             # the slow warpgroup sits out this step
        try:
            waits[k] = next(agents[k])
        except StopIteration:
            live.discard(k)
    assert all(r == set(range(8)) for r in a_rel + b_rel), "entries left unreleased at the end"


def _generator_plans():
    for name, spec in MB.LAYERS:
        n_tile = spec.get("n_tile") or (128 if (4 * spec["cout"] if spec["kind"] == "merged" else spec["cout"]) % 128 == 0
                                        else 64)
        for split in ((1,) if spec["kind"] == "rowk" else (2, 1, 0)):
            for li, geo in enumerate(plan_geometry(spec, n_tile, split)):
                yield pytest.param(geo, id="%s-split%d-launch%d" % (name.split(" @")[0].replace(" ", "_"), split, li))


@pytest.mark.parametrize("geo", list(_generator_plans()))
def test_ring_protocol_with_a_delayed_warpgroup(geo):
    cnts, chunks, a_stages, b_stages = geo
    chunks = min(chunks, 3)                      # the protocol repeats per chunk; three keep the run short
    for seed in range(4):
        simulate(cnts, chunks, a_stages, b_stages, tiles=3, seed=seed, slow_wg=seed % 2)
