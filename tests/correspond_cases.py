"""Seeded cases of the rasterizer front-ends, registered in glue_cases.CASES / REQUIRED_EDGES (so test_glue_kernels_gpu.py
runs them on the kernels and test_glue_cases_cpu.py the correspondence cases on kernel_emulator):

* ``correspond`` (lwb_correspond: raster + cond + T + source-image warp in one pass), every output a caller buffer;
* ``raster_forward_face_index_map`` (the nr.rasterize mirror, GPU only) on caller pre-filled maps.

The checks compare with restatements, never with the emulator: f2verts with oracle.nmr_ref.project_to_faces (pinned to the
reference code by tests/golden/make_nmr_golden.py), fim / wim / depth / faces_inv with the C restatement of the reference
rasterizer (oracle/raster_ref.c), cond with map_fn[fim], T and the warped image with float64 sums.  The inputs and the
oracle's rasterization are built at the first use, not at import.
"""
import torch
import torch.nn.functional as F

from glue_cases import Bits, Case, Tol, NAN, _gen, _pin_nan

NEAR, FAR = 0.1, 100.0
FIM_FILL, DEPTH_FILL, INV_FILL = -12345, NAN, 7.0          # raster_forward prefills: uncovered pixels keep them


def _canon(t):
    """+0.0 for -0.0 (NaN kept): the sign of a zero weight or coordinate is not part of the contract -- the C
    restatement's clamp and torch's identity matmul in look_at may each give the other zero than the kernel."""
    return t + 0.0


def _memo(build):
    cache = []

    def get():
        if not cache:
            cache.append(build())
        return cache[0]
    return get


# ----------------------------------------------------------------------------------------------------------- meshes
def _mesh(kind):
    from impersonator_b200 import synthetic as S
    if kind == "sphere":                                  # the SMPL-sized sphere of bench.py: V = 6890, F = 13776
        return S.uv_sphere()
    if kind == "small":                                   # V = 146, F = 288
        return S.uv_sphere(rings=12, segments=12)
    n = int(kind[len("sheet"):])                          # an n x n vertex grid facing the camera, gently curved
    xs = torch.linspace(-0.95, 0.95, n)
    y, x = torch.meshgrid(xs, xs, indexing="ij")
    v = torch.stack([x, y, 0.05 * torch.sin(3 * x) * torch.cos(2 * y)], dim=-1).reshape(-1, 3)
    f = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, c = i * n + j, (i + 1) * n + j
            f += [(a, a + 1, c), (a + 1, c + 1, c)]
    return v.float(), torch.tensor(f, dtype=torch.int32)


def _back_facing(faces):
    """rasterize_cuda_kernel.cu:57 in fp32 (each torch CPU operation rounds once, as the C restatement and the kernel)."""
    f = faces.reshape(faces.shape[0], faces.shape[1], 9)
    return (f[..., 7] - f[..., 1]) * (f[..., 3] - f[..., 0]) < (f[..., 4] - f[..., 1]) * (f[..., 6] - f[..., 0])


def _frames(seed, B, v, f, sheet_facing=None):
    """-> cam [B,3], verts [B,V,3], face_idx [F,3]; a sheet keeps its pose (cameras vary) and is wound so that every
    face is front-facing (sheet_facing="front") or back-facing ("back")."""
    from impersonator_b200 import synthetic as S
    from oracle import nmr_ref
    if sheet_facing is None:
        cam, verts = S.synthetic_frames(B, seed=seed, base_verts=v)
        return cam, verts, f
    g = _gen(seed)
    cam = torch.cat([0.9 + 0.2 * torch.rand(B, 1, generator=g), (torch.rand(B, 2, generator=g) - 0.5) * 0.1], dim=1)
    verts = v[None].repeat(B, 1, 1).contiguous()
    back = _back_facing(nmr_ref.project_to_faces(cam, verts, f))
    if bool(back.all()) != (sheet_facing == "back"):
        f = f[:, [0, 2, 1]].contiguous()
        back = _back_facing(nmr_ref.project_to_faces(cam, verts, f))
    assert bool(back.all()) == (sheet_facing == "back") and bool(back.any()) == (sheet_facing == "back")
    return cam, verts, f


# ------------------------------------------------------------------------------------------------------- correspond
def _correspond(edge, seed, B, s, mesh="small", sb=1, ac=1, C=3, src_img=True, near=NEAR, far=FAR, sheet=None,
                frames=None, source=None, dup=False):
    """frames(cam, verts): edits the target frames in place; source: "off-screen" (source cameras scaled 3x: the
    tables reach |p2v| ~ 2.7) | "only_vis" (get_vis_f2pts of the source's own rasterization: -2 rows); dup: every face
    twice (face i and face 2F-1-i), depth ties the lowest index wins."""
    def build():
        from oracle import nmr_ref, raster
        g = _gen(seed)
        v, f = _mesh(mesh)
        cam, verts, f = _frames(seed, B, v, f, sheet)
        if dup:
            f = torch.cat([f, f.flip(0)]).contiguous()
        if frames is not None:
            frames(cam, verts)
        nf = f.shape[0]
        cam_s, verts_s, _ = _frames(seed + 1, sb, v, f, sheet)
        if source == "off-screen":
            cam_s[:, 0] *= 3.0
        faces_s = nmr_ref.project_to_faces(cam_s, verts_s, f)
        p2v = nmr_ref.src_p2verts(faces_s).contiguous()
        if source == "only_vis":
            fim_s = torch.from_numpy(raster.rasterize_fim_wim(faces_s.numpy(), s)[0])
            p2v = nmr_ref.get_vis_f2pts(p2v, fim_s).contiguous()
            assert bool((p2v == -2).all(dim=(2, 3)).any()) and not bool((p2v == -2).all())
        img = torch.rand(sb, 3, s, s, generator=g) * 2 - 1 if src_img else None
        map_fn = torch.rand(nf + 1, C, generator=g) * 2 - 1                  # background row F unlike row 0
        return dict(cam=cam, verts=verts, f=f, p2v=p2v, img=img, map_fn=map_fn, nf=nf)
    inputs = _memo(build)

    def refs_build():
        from oracle import nmr_ref, raster
        i = inputs()
        faces = nmr_ref.project_to_faces(i["cam"], i["verts"], i["f"])
        fim, wim, _ = raster.rasterize_fim_wim(faces.numpy(), s, near, far)
        fim, wim = torch.from_numpy(fim), torch.from_numpy(wim)
        cov = fim >= 0
        q = i["p2v"].double().expand(B, -1, -1, -1)
        pts = q[torch.arange(B)[:, None, None], fim.long().clamp(min=0)]               # [B,s,s,3,2]
        terms = wim.double()[..., None] * pts
        return dict(faces=faces, fim=fim, wim=wim, cov=cov, cond=nmr_ref.encode_fim(fim, i["map_fn"]).contiguous(),
                    T=terms.sum(3)[cov], ST=terms.abs().sum(3)[cov])
    refs = _memo(refs_build)

    def warp64(o):
        """grid_sample(src, T) in float64 at the kernel's own T, and its S in units of u.  The bilinear sum of four taps
        rounds its tap weights, products and adds: a few u on the same sample of |src|.  The kernel's fp32
        un-normalisation ((T + 1) / 2 * (s - 1), or ((T + 1) s - 1) / 2) puts the sample point up to about
        2 u s (1 + |T|) + u pixels off along each axis, and the bilinear surface (zero padded) has a slope of at most
        2 max|src| per pixel: together 4 u max|src| (s (2 + |Tx| + |Ty|) + 1)."""
        i = inputs()
        src = i["img"].double() if i["img"] is not None else torch.zeros(1, 3, s, s, dtype=torch.float64)
        src = src.expand(B, -1, -1, -1)
        T = o["T"].double()
        val = F.grid_sample(src, T, mode="bilinear", padding_mode="zeros", align_corners=bool(ac))
        mag = F.grid_sample(src.abs(), T, mode="bilinear", padding_mode="zeros", align_corners=bool(ac))
        coord = 4 * (s * (2 + T.abs().sum(-1)) + 1)[:, None] * src.abs().amax(dim=(1, 2, 3))[:, None, None, None]
        return val, mag + coord

    def run(api, put, alloc):
        i = inputs()
        C_ = i["map_fn"].shape[1]
        o = dict(fim=alloc(torch.full((B, s, s), FIM_FILL, dtype=torch.int32)), wim=alloc(torch.full((B, s, s, 3), NAN)),
                 T=alloc(torch.full((B, s, s, 2), NAN)), tsf_inputs=alloc(torch.full((B, 3 + C_, s, s), NAN)),
                 f2verts=alloc(torch.full((B, i["nf"], 3, 3), NAN)))
        cam, verts, f, map_fn, p2v, img = (put(t) if t is not None else None for t in (
            i["cam"], i["verts"], i["f"], i["map_fn"], i["p2v"], i["img"]))
        api.correspond(cam, verts, f, s, map_fn, p2v, img, align_corners=bool(ac), want_f2verts=True, near=near, far=far,
                       out=o)
        return {k: o[k] for k in ("fim", "wim", "T", "tsf_inputs", "f2verts")}

    checks = [
        Bits("f2verts", lambda o: _canon(o["f2verts"]), lambda o: _pin_nan(_canon(o["f2verts"]), _canon(refs()["faces"]))),
        Bits("fim", "fim", lambda o: refs()["fim"]),
        Bits("wim", lambda o: _canon(o["wim"]), lambda o: _canon(refs()["wim"])),
        Bits("cond (tsf_inputs[:, 3:])", lambda o: o["tsf_inputs"][:, 3:], lambda o: refs()["cond"]),
        Bits("T background", lambda o: o["T"][~refs()["cov"]], lambda o: torch.full((int((~refs()["cov"]).sum()), 2), -2.0)),
        Tol("T covered", lambda o: o["T"][refs()["cov"]], lambda: refs()["T"], lambda: refs()["ST"], 3),
        Tol("tsf_img (tsf_inputs[:, :3])", lambda o: o["tsf_inputs"][:, :3], lambda o: warp64(o)[0], lambda o: warp64(o)[1],
            4, of_outputs=True),
    ]
    case = Case("correspond", edge, run, checks)
    case.inputs, case.refs = inputs, refs
    return case


def _off_screen(*frames):
    def edit(cam, verts):
        for b in frames:
            cam[b, 1] = 5.0                                   # translated 5 NDC units to the side: nothing on screen
    return edit


def _nan_frame(cam, verts):
    verts[1] = NAN


def _zero(cam, verts):
    verts.zero_()


def correspond_cases():
    return [
        _correspond("sphere 256 B=3 sb=1 ac=0", 2001, 3, 256, mesh="sphere", ac=0),
        _correspond("sphere 256 B=3 sb=1 ac=1", 2002, 3, 256, mesh="sphere", ac=1),
        _correspond("sphere 512 B=1", 2003, 1, 512, mesh="sphere"),
        _correspond("size 1", 2004, 2, 1, frames=_off_screen(1)),           # ac=1: the background samples src[0, 0]
        _correspond("size 2 ac=1", 2005, 2, 2, mesh="sheet5", sheet="front", frames=_off_screen(1)),  # background: src[0, 0] / 4
        _correspond("size 33 B=5", 2006, 5, 33),
        _correspond("size 300", 2007, 2, 300, ac=0),
        _correspond("sb=B", 2008, 3, 64, sb=3),
        _correspond("src_img None", 2009, 2, 64, src_img=False),
        _correspond("map_c=1", 2010, 2, 48, C=1),
        _correspond("map_c=5", 2011, 2, 48, C=5),
        _correspond("off-screen source", 2012, 2, 64, source="off-screen", sb=2),
        _correspond("only_vis tables", 2013, 2, 64, source="only_vis"),
        _correspond("frame off screen", 2014, 2, 40, frames=_off_screen(0, 1)),
        _correspond("NaN frame", 2015, 3, 64, frames=_nan_frame),
        _correspond("all back-facing", 2016, 2, 64, mesh="sheet9", sheet="back"),
        _correspond("near plane crossing", 2017, 2, 64, near=2.62, far=2.85),
        _correspond("all-zero vertices", 2018, 2, 64, frames=_zero),
        _correspond("big faces", 2019, 2, 128, mesh="sheet3", sheet="front"),
        _correspond("duplicate faces", 2020, 2, 64, dup=True),
        _correspond("B=17", 2021, 17, 40),
    ]


CORRESPOND_EDGES = [
    "sphere 256 B=3 sb=1 ac=0", "sphere 256 B=3 sb=1 ac=1", "sphere 512 B=1", "size 1", "size 2 ac=1", "size 33 B=5",
    "size 300", "sb=B", "src_img None", "map_c=1", "map_c=5", "off-screen source", "only_vis tables", "frame off screen",
    "NaN frame", "all back-facing", "near plane crossing", "all-zero vertices", "big faces", "duplicate faces", "B=17"]


# --------------------------------------------------------------------------------------- raster_forward_face_index_map
def _raster(edge, seed, B, s, depth=True, faces_inv=True, flip=False, near=NEAR, far=FAR, frames=None):
    def build():
        from oracle import nmr_ref
        v, f = _mesh("small")
        cam, verts, f = _frames(seed, B, v, f)
        if frames is not None:
            frames(cam, verts)
        return nmr_ref.project_to_faces(cam, verts, f).contiguous()
    faces = _memo(build)

    def want_build():
        from oracle import raster
        fc = faces()
        fim, wim, dep, inv = (torch.from_numpy(a) for a in raster.forward_face_index_map_cpu(fc.numpy(), s, near, far))
        cov = fim >= 0
        w = dict(fim=torch.where(cov, fim, torch.tensor(FIM_FILL, dtype=torch.int32)),
                 wim=torch.where(cov[..., None], wim, torch.tensor(NAN)),
                 depth=torch.where(cov, dep, torch.tensor(DEPTH_FILL)),
                 faces_inv=torch.where(_back_facing(fc)[..., None, None], torch.tensor(INV_FILL), inv))
        if flip:
            for k in ("fim", "wim", "depth"):
                w[k] = w[k].flip(1)
        assert 0 < int(cov.sum()) < cov.numel()
        return {k: t.contiguous() for k, t in w.items()}
    want = _memo(want_build)

    def run(api, put, alloc):
        fc = faces()
        nf = fc.shape[1]
        o = dict(fim=alloc(torch.full((B, s, s), FIM_FILL, dtype=torch.int32)), wim=alloc(torch.full((B, s, s, 3), NAN)))
        if depth:
            o["depth"] = alloc(torch.full((B, s, s), DEPTH_FILL))
        if faces_inv:
            o["faces_inv"] = alloc(torch.full((B, nf, 3, 3), INV_FILL))
        api.raster_forward_face_index_map(put(fc), o["fim"], o["wim"], o.get("depth"), s, near=near, far=far,
                                          faces_inv=o.get("faces_inv"), flip_rows=flip)
        return o

    checks = [Bits("fim", "fim", lambda o: want()["fim"]),
              Bits("wim", lambda o: _canon(o["wim"]), lambda o: _canon(want()["wim"]))]
    if depth:
        checks.append(Bits("depth", "depth", lambda o: want()["depth"]))
    if faces_inv:
        checks.append(Bits("faces_inv", "faces_inv", lambda o: want()["faces_inv"]))
    return Case("raster_forward_face_index_map", edge, run, checks, emulated=False)


def raster_cases():
    return [
        _raster("sphere 128 B=2", 2101, 2, 128),
        _raster("prefill kept", 2102, 3, 64, frames=lambda cam, verts: (cam[:, 0].mul_(0.3), cam[1, 1].fill_(5.0))),
        _raster("depth None", 2103, 2, 64, depth=False),
        _raster("faces_inv None", 2104, 2, 64, faces_inv=False),
        _raster("flip_rows", 2105, 2, 64, flip=True),
        _raster("near far custom", 2106, 2, 64, near=2.62, far=2.85),
        _raster("size 33 B=3", 2107, 3, 33),
    ]


RASTER_EDGES = ["sphere 128 B=2", "prefill kept", "depth None", "faces_inv None", "flip_rows", "near far custom",
                "size 33 B=3"]
