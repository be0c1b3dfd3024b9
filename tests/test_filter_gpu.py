"""The 2-D screen-space filter on the fused frame path (gs_ctx_set_filter2d, RenderContext.set_filter2d,
`Splatter(..., filter2d=...)`) against the fp64 oracle of tests/filter_oracle.py: every blend kernel family (RGB, scalar
and tensor-core per-pixel SH, per-Gaussian SH, aux maps, the packed path), camera gradients, a single Gaussian's
screen-space integral, the mode's lifetime on a context, the data-parallel push routing and the full C3 size."""
import pytest
import torch

import filter_oracle as F
import gs_oracle as O
import sh_gaussian_oracle as G
import synthetic as S
from helpers import abs_err, device_depth_keys, rel_err, scene
from test_scale_parity_gpu import _pick_tiles, _tile_mask

pytestmark = pytest.mark.gpu

IMG_ATOL = 1e-4
GRAD_RTOL = 1e-3
BG = (0.2, 0.5, 0.9)
NAMES = ("pos", "rgb", "opa", "quat", "scale")
MODES = ["dilate", "antialias"]
# colour model: (colour width, sh_eval, sh_tc knob or None)
COLOURS = {"rgb": (3, "pixel", None), "sh27-tc0": (27, "pixel", 0), "sh27-tc3": (27, "pixel", 3),
           "sh48-tc0": (48, "pixel", 0), "sh48-tc3": (48, "pixel", 3), "sh27-gauss": (27, "gaussian", None),
           "sh48-gauss": (48, "gaussian", None)}


def _args(v):
    return (v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")


def _splatter(g, v, dev, **kw):
    import splatter
    vs = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)]
    return splatter.Splatter.from_tensors(g, vs, device=dev, use_sh_coeff=g["rgb"].shape[1] != 3, **kw)


def _ctx(gs, mode, sh_eval="pixel", variance=0.3):
    import renderer
    rctx = gs[0].RenderContext()
    rctx.set_sh_eval(renderer.SH_EVAL[sh_eval])
    rctx.set_filter2d(renderer.FILTER2D[mode], variance)
    return rctx


def _colour(p, cam, sh_eval):
    """(rgb argument, use_sh_coeff) of the oracle for the colour model of the frame."""
    if p["rgb"].shape[1] == 3:
        return p["rgb"], False
    if sh_eval == "gaussian":
        return G.gaussian_logits(p["pos"], p["rgb"], cam), False
    return p["rgb"], True


def _upstream(rows, cols, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(rows, cols, 3, generator=gen, dtype=torch.float64) * 2 - 1


def _check_grads(got, ref, label=""):
    for q in NAMES:
        g = got[q]
        assert bool(torch.isfinite(g).all()), (label, q)
        assert rel_err(g, ref[q]) < GRAD_RTOL, (label, q, rel_err(g, ref[q]))


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("colour", list(COLOURS))
@pytest.mark.parametrize("mode", MODES)
def test_filter_frame_vs_oracle(gs, cuda, mode, colour, final):
    """Splatter.forward (final) and Splatter.render_padded (padded) with the filter against the oracle: image 1e-4 abs,
    all five gradients 1e-3 relative, for every blend kernel family."""
    sh_dim, sh_eval, tc = COLOURS[colour]
    n, w, h = (4000, 128, 96) if sh_dim == 3 else (2500, 112, 80)
    g, v, cam = scene(n, w, h, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    go = _upstream(h, w) if final else _upstream(cam.Hp, cam.Wp)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    rgb, use_sh = _colour(p, cam, sh_eval)
    img, aux = F.render(p["pos"], rgb, p["opa"], p["quat"], p["scale"], cam, mode, use_sh_coeff=use_sh,
                        return_aux=True, depth_key=device_depth_keys(g, cam, cuda))
    out = img if final else aux["padded"]
    out.backward(go)
    if tc is not None:
        gs[0].tune("sh_tc", tc)
    try:
        sp = _splatter(g, v, cuda, sh_eval=sh_eval, filter2d=mode)
        if final:
            got = sp(0)
        else:
            sp.set_camera(0)
            got = sp.render_padded()
        got.backward(go.float().to(cuda))
        torch.cuda.synchronize()
    finally:
        gs[0].tune("sh_tc", -1)
    assert abs_err(got, out) < IMG_ATOL
    _check_grads({q: getattr(sp.gaussian_3ds, q).grad for q in NAMES}, {q: p[q].grad for q in NAMES})


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("mode", MODES)
def test_filter_aux_vs_oracle(gs, cuda, mode, final):
    """Depth / alpha maps over a background (Splatter.render_maps for the final maps, renderer.render_frame_aux for the
    padded ones) under depth-only and alpha-only upstream gradients."""
    import renderer
    g, v, cam = scene(4000, 128, 96, k=1, opa_range=(0.05, 0.9))
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    o = F.render_maps(*(p[q] for q in NAMES), cam, mode, background=BG, depth_key=device_depth_keys(g, cam, cuda))
    oi, od, oa = (o["image"], o["depth"], o["alpha"]) if final else (o["padded_image"], o["padded_depth"],
                                                                      o["padded_alpha"])
    dmax = float(od.detach().abs().max())
    gen = torch.Generator().manual_seed(5)
    gd = torch.rand(od.shape, generator=gen, dtype=torch.float64) * 2 - 1
    ga = torch.rand(od.shape, generator=gen, dtype=torch.float64) * 2 - 1
    sp = _splatter(g, v, cuda, filter2d=mode)
    rctx = _ctx(gs, mode)
    for case, (which, upstream) in {"depth": (od, gd), "alpha": (oa, ga)}.items():
        ref = torch.autograd.grad(which, [p[q] for q in NAMES], upstream, retain_graph=True, allow_unused=True)
        if final:
            for q in NAMES:
                getattr(sp.gaussian_3ds, q).grad = None
            m = sp.render_maps(0, background=BG)
            img, dep, alp = m["image"], m["depth"], m["alpha"]
            params = {q: getattr(sp.gaussian_3ds, q) for q in NAMES}
        else:
            params = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
            img, dep, alp, _ = renderer.render_frame_aux(rctx, *(params[q] for q in NAMES), *_args(v), background=BG,
                                                         final=False)
        assert abs_err(img, oi) < IMG_ATOL
        assert abs_err(alp, oa) < 1e-4
        assert abs_err(dep, od) < 1e-4 * dmax
        (dep if case == "depth" else alp).backward(upstream.float().to(cuda))
        _check_grads({q: params[q].grad for q in NAMES},
                     {q: torch.zeros_like(p[q]) if r is None else r for q, r in zip(NAMES, ref)}, case)


@pytest.mark.parametrize("mode", MODES)
def test_filter_packed_path_vs_oracle(gs, cuda, mode):
    """The packed path (gs_tune("gather", 0)): pack_sorted and the packed RGB blend kernels."""
    g, v, cam = scene(4000, 128, 96, k=1, opa_range=(0.05, 0.9))
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    oimg = F.render(*(p[q] for q in NAMES), cam, mode, depth_key=device_depth_keys(g, cam, cuda))
    go = _upstream(96, 128)
    oimg.backward(go)
    gs[0].tune("gather", 0)
    try:
        sp = _splatter(g, v, cuda, filter2d=mode)
        img = sp(0)
        img.backward(go.float().to(cuda))
        torch.cuda.synchronize()
    finally:
        gs[0].tune("gather", 1)
    assert abs_err(img, oimg) < IMG_ATOL
    _check_grads({q: getattr(sp.gaussian_3ds, q).grad for q in NAMES}, {q: p[q].grad for q in NAMES})


@pytest.mark.parametrize("params_grad", [True, False], ids=["params+pose", "pose"])
@pytest.mark.parametrize("sh_dim", [3, 48])
def test_filter_cam_grad_vs_oracle(gs, cuda, sh_dim, params_grad):
    """gs_render_backward_cam of an antialiased frame (image + depth upstream over a background): dL/drot, dL/dtran
    (and the parameter gradients) against oracle autograd; camera only when no parameter needs a gradient."""
    import renderer
    sh_eval = "gaussian" if sh_dim != 3 else "pixel"
    g, v, cam = scene(4000, 128, 96, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    rot, tran = v.rot.double().clone().requires_grad_(True), v.tran.double().clone().requires_grad_(True)
    ocam = O.Camera(v.width, v.height, v.fx, v.fy, rot, tran, v.near)
    rgb, _ = _colour(p, ocam, sh_eval)
    o = F.render_maps(p["pos"], rgb, p["opa"], p["quat"], p["scale"], ocam, "antialias", background=BG,
                      depth_key=device_depth_keys(g, cam, cuda))
    gen = torch.Generator().manual_seed(7)
    gi = torch.rand(o["image"].shape, generator=gen, dtype=torch.float64) * 2 - 1
    gd = (torch.rand(o["depth"].shape, generator=gen, dtype=torch.float64) * 2 - 1) * 1e-2
    ref = torch.autograd.grad([o["image"], o["depth"]], [p[q] for q in NAMES] + [rot, tran], [gi, gd])
    rctx = _ctx(gs, "antialias", sh_eval)
    d = {q: t.to(cuda).clone().requires_grad_(params_grad) for q, t in g.items()}
    drot, dtran = v.rot.to(cuda).requires_grad_(True), v.tran.to(cuda).requires_grad_(True)
    img, dep, _, _ = renderer.render_frame_cam(rctx, *(d[q] for q in NAMES), v.width, v.height, v.fx, v.fy, drot,
                                               dtran, v.near, 0.05, "abs", background=BG)
    torch.autograd.backward([img, dep], [gi.float().to(cuda), gd.float().to(cuda)])
    assert abs_err(img, o["image"]) < IMG_ATOL
    assert rel_err(drot.grad, ref[5]) < GRAD_RTOL, rel_err(drot.grad, ref[5])
    assert rel_err(dtran.grad, ref[6]) < GRAD_RTOL, rel_err(dtran.grad, ref[6])
    if params_grad:
        _check_grads({q: d[q].grad for q in NAMES}, dict(zip(NAMES, ref)))


def test_single_gaussian_screen_space_integral(gs, cuda):
    """One centred Gaussian, sigma = 3 px, opacity 0.01, 32 x 32, variance 0.3: antialias keeps the alpha-map sum of the
    unfiltered frame, dilate raises it by (9 + 0.3) / 9."""
    import renderer
    fx = fy = 40.0
    z = 5.0
    g = dict(pos=torch.tensor([[0.0, 0.0, z]]), rgb=torch.zeros(1, 3), opa=torch.tensor([-4.59511985013459]),
             quat=torch.tensor([[1.0, 0.0, 0.0, 0.0]]), scale=torch.full((1, 3), 3.0 * z / fx - 1e-4))
    d = {q: t.to(cuda) for q, t in g.items()}
    sums = {}
    for mode in ("none", "dilate", "antialias"):
        rctx = _ctx(gs, mode)
        _, _, alp, _ = renderer.render_frame_aux(rctx, *(d[q] for q in NAMES), 32, 32, fx, fy, torch.eye(3),
                                                 torch.zeros(3), 0.3, 0.05, "abs", final=False)
        sums[mode] = float(alp.double().sum())
    assert abs(sums["antialias"] / sums["none"] - 1) <= 1e-3, sums
    assert abs(sums["dilate"] / sums["none"] - 9.3 / 9) <= 1e-3, sums


def test_mode_belongs_to_the_forward(gs, cuda):
    """Mode none with a variance set is bit-identical to a context that never called the setter; changing the setting
    between forward and backward leaves that backward's gradients unchanged bit for bit; bad settings are refused."""
    import renderer
    g, v, cam = scene(4000, 128, 96, k=1, opa_range=(0.05, 0.9))
    go = _upstream(96, 128).float().to(cuda)

    def frame(rctx, switch_to=None):
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        img, _ = renderer.render_frame_final(rctx, *(d[q] for q in NAMES), *_args(v))
        if switch_to is not None:
            rctx.set_filter2d(renderer.FILTER2D[switch_to], 2.0)
        img.backward(go)
        return [img.detach()] + [d[q].grad for q in NAMES]

    fresh = frame(gs[0].RenderContext())
    for a, b in zip(fresh, frame(_ctx(gs, "none", variance=1.7))):
        assert torch.equal(a, b)
    for mode, other in (("antialias", "none"), ("dilate", "antialias"), ("none", "dilate")):
        plain = frame(_ctx(gs, mode))
        switched = frame(_ctx(gs, mode), switch_to=other)
        for a, b in zip(plain, switched):
            assert torch.equal(a, b), mode
    filtered = frame(_ctx(gs, "antialias"))
    assert not torch.equal(filtered[0], fresh[0])
    rctx = gs[0].RenderContext()
    for mode, var in ((-1, 0.3), (3, 0.3), (1, 0.0), (2, -1.0), (0, float("nan")), (1, float("inf"))):
        with pytest.raises(RuntimeError, match="gs_ctx_set_filter2d"):
            rctx.set_filter2d(mode, var)
    for kw in (dict(filter2d="mip"), dict(filter2d="dilate", filter2d_variance=0.0),
               dict(filter2d="antialias", filter2d_variance=float("nan")), dict(filter2d_variance="x")):
        with pytest.raises(ValueError, match="filter2d"):
            _splatter(g, v, cuda, **kw)


@pytest.mark.parametrize("rank", [0, 1])
def test_push_routing_on_one_gpu(gs, cuda, rank):
    """Data-parallel push with world = 2 and both staging buffers on this device, antialias: the bucket's own slice plus
    the slot this rank wrote into the other owner's staging buffer reproduce the non-push gradients bit for bit."""
    import renderer
    g, v, cam = scene(4000, 128, 96, k=1, opa_range=(0.05, 0.9))
    go = _upstream(96, 128).float().to(cuda)
    world = 2
    made = {}

    def run(push):
        def alloc(numel, device):
            per = (numel + world * 4 - 1) // (world * 4) * 4
            flat = torch.zeros(world * per, device=device)
            made["flat"], made["per"], made["numel"] = flat, per, numel
            if not push:
                return flat
            made["staging"] = [torch.full((world * per,), float("nan"), device=device) for _ in range(world)]
            return flat, (flat.data_ptr(), [s.data_ptr() for s in made["staging"]], per, rank)

        rctx = _ctx(gs, "antialias")
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        renderer.set_flat_grad_allocator(alloc)
        try:
            img, _ = renderer.render_frame_final(rctx, *(d[q] for q in NAMES), *_args(v))
            img.backward(go)
        finally:
            renderer.set_flat_grad_allocator(None)
        torch.cuda.synchronize()
        return dict(made)

    ref = run(False)
    got = run(True)
    per, numel = got["per"], got["numel"]
    other = 1 - rank
    mine = got["flat"][rank * per:(rank + 1) * per]
    theirs = got["staging"][other][rank * per:(rank + 1) * per]
    joined = torch.cat([mine, theirs] if rank == 0 else [theirs, mine])[:numel]
    assert torch.equal(joined, ref["flat"][:numel])


def test_c3_antialias_properties_and_masked_parity(gs, cuda):
    """C3 (2.4 M Gaussians, 1080p) with antialias: bit-deterministic, as many launches as the unfiltered frame, M close
    to the CPU oracle's 7,354,944 instances, and fp64 oracle parity on sampled tiles (upstream gradient non-zero only
    there; every other gradient exactly 0)."""
    import renderer
    n, w, h = 2_400_000, 1920, 1080
    g = S.make_gaussians(n, w, h, 0)
    v = S.make_view(w, h, 0)
    cam = O.Camera(w, h, v.fx, v.fy, v.rot, v.tran, v.near)
    go = (torch.rand(h, w, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1).to(cuda)
    dev = {q: t.to(cuda) for q, t in g.items()}

    def frame(rctx):
        d = {q: t.clone().requires_grad_(True) for q, t in dev.items()}
        l0 = gs[0].kernel_launches()
        img, _ = renderer.render_frame_final(rctx, *(d[q] for q in NAMES), *_args(v))
        img.backward(go)
        torch.cuda.synchronize()
        return [img.detach()] + [d[q].grad for q in NAMES], gs[0].kernel_launches() - l0, rctx.stats()

    rctx = _ctx(gs, "antialias")
    frame(rctx)                                            # the first frame of a context also fills its index table
    a, la, sa = frame(rctx)
    b, lb, _ = frame(rctx)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    del a, b
    r0 = _ctx(gs, "none")
    frame(r0)
    _, l0, s0 = frame(r0)
    del r0
    assert la == lb == l0
    m_cpu = 7_354_944
    print(f"\nC3 antialias: M = {sa['n_instances']} (CPU oracle {m_cpu}, difference {sa['n_instances'] - m_cpu}); "
          f"unfiltered M = {s0['n_instances']}; M_eff = {sa['n_instances_eff']} (unfiltered {s0['n_instances_eff']})")
    assert abs(sa["n_instances"] - m_cpu) <= 1e-4 * m_cpu
    del dev

    sp = _splatter(g, v, cuda, filter2d="antialias")
    with torch.no_grad():
        sp(0)
    idx, accum = sp._rctx.sorted_instances()
    idx, accum = idx.cpu(), accum.cpu().long()
    neff = sp._rctx.tile_consumed().cpu().long()
    tiles = _pick_tiles(accum, neff, cam.ntx, cam.nty, 5)
    top, left = (cam.Hp - h) // 2, (cam.Wp - w) // 2
    gom = S.make_grad_output(h, w, 0) * (h * w) * _tile_mask(cam, tiles, h, w)
    img = sp(0)
    img.backward(gom.to(cuda))
    opad, U, ograds = _oracle_on_tiles(g, cam, idx, accum, tiles, gom)
    raw = torch.zeros(cam.Hp, cam.Wp, 3, dtype=torch.float64)
    raw[top:top + h, left:left + w] = img.detach().cpu().double()
    for t in tiles:
        ty, tx = divmod(t, cam.ntx)
        r0_, r1_ = max(ty * 16, top), min((ty + 1) * 16, top + h)
        assert abs_err(raw[r0_:r1_, tx * 16:(tx + 1) * 16], opad[r0_:r1_, tx * 16:(tx + 1) * 16].clamp(0, 1)) < IMG_ATOL
    other = torch.ones(n, dtype=torch.bool)
    other[U] = False
    for q in NAMES:
        got = getattr(sp.gaussian_3ds, q).grad.cpu()
        assert bool(torch.isfinite(got).all()), q
        assert rel_err(got[U], ograds[q]) < GRAD_RTOL, q
        assert float(got[other].abs().max()) == 0.0, q


def _oracle_on_tiles(g, cam, idx, accum, tiles, go_final):
    """fp64 antialias oracle restricted to the Gaussians the DEVICE binned into `tiles`, in the device's order (binning
    and order parity are checked elsewhere).  Returns (padded image, U, gradients on U)."""
    dt = torch.float64
    ids = [idx[int(accum[t]):int(accum[t + 1])].long() for t in tiles]
    U = torch.unique(torch.cat(ids))
    p = {k: g[k][U].to(dt).clone().requires_grad_(True) for k in NAMES}
    nq, ns, opa_a, rgb_a = O.preactivate(p["quat"], p["scale"], p["opa"], p["rgb"])
    rp, rc, _ = O.global_culling(p["pos"], nq, ns, cam.rot.to(dt), cam.tran.to(dt), cam.near, cam.half_w, cam.half_h)
    rcf, opf, _ = F.filtered(rc, opa_a, cam, "antialias")
    loc = torch.cat([torch.searchsorted(U, i) for i in ids])
    counts = torch.zeros(cam.ntx * cam.nty, dtype=torch.int64)
    for t, i in zip(tiles, ids):
        counts[t] = i.numel()
    acc2 = torch.zeros(cam.ntx * cam.nty + 1, dtype=torch.int64)
    acc2[1:] = torch.cumsum(counts, 0)
    padded = O.draw(rp[loc], rgb_a[loc], opf[loc], rcf[loc], acc2.to(torch.int32), cam.Hp, cam.Wp, cam.fx, cam.fy,
                    tiles=torch.tensor(tiles))
    cam.crop(torch.clamp(padded, 0, 1)).backward(go_final.to(dt))
    return padded.detach(), U, {k: p[k].grad for k in NAMES}
