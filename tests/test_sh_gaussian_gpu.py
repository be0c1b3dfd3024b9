"""SH colour evaluated once per Gaussian on the fused frame path (gs_ctx_set_sh_eval(ctx, GS_SH_EVAL_GAUSSIAN),
`Splatter(..., sh_eval="gaussian")`) against the fp64 oracle of tests/sh_gaussian_oracle.py: plain and aux frames,
the packed path, agreement with the per-pixel kernels where the two models coincide, the mode's lifetime on a
context, the data-parallel push routing and the full C3 size."""
import pytest
import torch

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
# the C1-class scenes of the per-pixel SH frame tests (test_frame_gpu.py): (colour width, opacity range)
SCENES = [(27, (0.005, 0.05)), (27, (0.3, 0.95)), (48, (0.05, 0.9))]
SCENE_IDS = ["sh27-safe", "sh27-opaque", "sh48"]


def _args(v):
    return (v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")


def _splatter(g, v, dev, **kw):
    import splatter
    vs = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)]
    return splatter.Splatter.from_tensors(g, vs, device=dev, use_sh_coeff=g["rgb"].shape[1] != 3, **kw)


def _ctx(gs, mode):
    import renderer
    rctx = gs[0].RenderContext()
    rctx.set_sh_eval(renderer.SH_EVAL[mode])
    return rctx


def _oracle(g, cam, cuda, go, final, maps=False, **kw):
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    key = device_depth_keys(g, cam, cuda)
    if maps:
        o = G.render_maps(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, depth_key=key, **kw)
        return o, p
    img, aux = G.render(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], cam, return_aux=True, depth_key=key)
    out = img if final else aux["padded"]
    out.backward(go)
    return out.detach(), {q: p[q].grad for q in NAMES}


def _upstream(rows, cols, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return (torch.rand(rows, cols, 3, generator=gen, dtype=torch.float64) * 2 - 1)


def _check_grads(got, ref, label=""):
    for q in NAMES:
        g = got[q]
        assert bool(torch.isfinite(g).all()), (label, q)
        assert rel_err(g, ref[q]) < GRAD_RTOL, (label, q, rel_err(g, ref[q]))


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("sh_dim,opa", SCENES, ids=SCENE_IDS)
def test_sh_gaussian_frame_vs_oracle(gs, cuda, sh_dim, opa, final):
    """Splatter.forward (final) and Splatter.render_padded (padded) against the oracle: image 1e-4 abs, all five
    gradients 1e-3 relative."""
    n, w, h = 2500, 112, 80
    g, v, cam = scene(n, w, h, k=1, sh_dim=sh_dim, opa_range=opa)
    go = _upstream(h, w) if final else _upstream(cam.Hp, cam.Wp)
    oimg, ograds = _oracle(g, cam, cuda, go, final)
    sp = _splatter(g, v, cuda, sh_eval="gaussian")
    if final:
        img = sp(0)
    else:
        sp.set_camera(0)
        img = sp.render_padded()
    assert abs_err(img, oimg) < IMG_ATOL
    img.backward(go.float().to(cuda))
    _check_grads({q: getattr(sp.gaussian_3ds, q).grad for q in NAMES}, ograds)


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("sh_dim", [27, 48])
def test_sh_gaussian_aux_vs_oracle(gs, cuda, sh_dim, final):
    """Depth / alpha maps over a background (Splatter.render_maps for the final maps, renderer.render_frame_aux for the
    padded ones) under depth-only and alpha-only upstream gradients."""
    import renderer
    g, v, cam = scene(2500, 112, 80, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    o, p = _oracle(g, cam, cuda, None, final, maps=True, background=BG)
    oi, od, oa = (o["image"], o["depth"], o["alpha"]) if final else (o["padded_image"], o["padded_depth"],
                                                                      o["padded_alpha"])
    dmax = float(od.detach().abs().max())
    gen = torch.Generator().manual_seed(5)
    gd = (torch.rand(od.shape, generator=gen, dtype=torch.float64) * 2 - 1)
    ga = (torch.rand(od.shape, generator=gen, dtype=torch.float64) * 2 - 1)
    sp = _splatter(g, v, cuda, sh_eval="gaussian")
    rctx = _ctx(gs, "gaussian")
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


def test_sh_gaussian_packed_path_vs_oracle(gs, cuda):
    """The packed path (gs_tune("gather", 0)) runs the frame through pack_sorted and the packed RGB blend kernels."""
    g, v, cam = scene(2500, 112, 80, k=1, sh_dim=48, opa_range=(0.05, 0.9))
    go = _upstream(80, 112)
    oimg, ograds = _oracle(g, cam, cuda, go, True)
    gs[0].tune("gather", 0)
    try:
        sp = _splatter(g, v, cuda, sh_eval="gaussian")
        img = sp(0)
        img.backward(go.float().to(cuda))
    finally:
        gs[0].tune("gather", 1)
    assert abs_err(img, oimg) < IMG_ATOL
    _check_grads({q: getattr(sp.gaussian_3ds, q).grad for q in NAMES}, ograds)


@pytest.mark.parametrize("sh_dim", [27, 48])
def test_dc_only_matches_per_pixel_kernels(gs, cuda, sh_dim):
    """DC-only colour: the basis is constant, so the per-Gaussian frame equals the per-pixel frame of the default
    kernels (image; pos / opa / quat / scale and DC gradients)."""
    g, v, cam = scene(2500, 112, 80, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    K = sh_dim // 3
    rgb = g["rgb"].reshape(-1, 3, K).clone()
    rgb[:, :, 1:] = 0
    g["rgb"] = rgb.reshape(-1, sh_dim)
    go = _upstream(80, 112).float().to(cuda)
    out = {}
    for mode in ("pixel", "gaussian"):
        sp = _splatter(g, v, cuda, sh_eval=mode)
        img = sp(0)
        img.backward(go)
        grads = {q: getattr(sp.gaussian_3ds, q).grad for q in NAMES}
        grads["rgb"] = grads["rgb"].reshape(-1, 3, K)[:, :, 0]
        out[mode] = img.detach(), grads
    assert abs_err(out["gaussian"][0], out["pixel"][0]) < IMG_ATOL
    for q in NAMES:
        assert rel_err(out["gaussian"][1][q], out["pixel"][1][q]) < GRAD_RTOL, q


def test_mode_belongs_to_the_forward(gs, cuda):
    """Changing the setting between forward and backward does not change that backward; a d = 3 frame ignores the
    setting bit for bit; an unknown mode is refused."""
    import renderer
    g, v, cam = scene(2500, 112, 80, k=1, sh_dim=48, opa_range=(0.05, 0.9))
    g3, _, _ = scene(2500, 112, 80, k=1, sh_dim=3, opa_range=(0.05, 0.9))
    go = _upstream(80, 112).float().to(cuda)

    def frame(rctx, gg, switch_to=None):
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in gg.items()}
        img, _ = renderer.render_frame_final(rctx, *(d[q] for q in NAMES), *_args(v))
        if switch_to is not None:
            rctx.set_sh_eval(renderer.SH_EVAL[switch_to])
        img.backward(go)
        return [img.detach()] + [d[q].grad for q in NAMES]

    for mode, other in (("gaussian", "pixel"), ("pixel", "gaussian")):
        rctx = _ctx(gs, mode)
        plain = frame(rctx, g)
        rctx.set_sh_eval(renderer.SH_EVAL[mode])
        switched = frame(rctx, g, switch_to=other)
        for a, b in zip(plain, switched):
            assert torch.equal(a, b), mode
    ref = frame(_ctx(gs, "pixel"), g3)
    for a, b in zip(ref, frame(_ctx(gs, "gaussian"), g3)):
        assert torch.equal(a, b)
    rctx = _ctx(gs, "pixel")
    for bad in (-1, 2):
        with pytest.raises(RuntimeError, match="mode must be"):
            rctx.set_sh_eval(bad)
    with pytest.raises(ValueError, match="use_sh_coeff"):
        _splatter(g3, v, cuda, sh_eval="gaussian")
    with pytest.raises(ValueError, match="sh_eval"):
        _splatter(g, v, cuda, sh_eval="vertex")


@pytest.mark.parametrize("rank", [0, 1])
def test_push_routing_on_one_gpu(gs, cuda, rank):
    """Data-parallel push with world = 2 and both staging buffers on this device: the bucket's own slice plus the
    slot this rank wrote into the other owner's staging buffer reproduce the non-push gradients bit for bit."""
    import renderer
    g, v, cam = scene(2500, 112, 80, k=1, sh_dim=48, opa_range=(0.05, 0.9))
    go = _upstream(80, 112).float().to(cuda)
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

        rctx = _ctx(gs, "gaussian")
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
    assert 3 * 2500 < per < 51 * 2500            # the slice boundary cuts the coefficient gradients
    other = 1 - rank
    mine = got["flat"][rank * per:(rank + 1) * per]
    theirs = got["staging"][other][rank * per:(rank + 1) * per]   # slot `rank` of the other owner's staging buffer
    joined = torch.cat([mine, theirs] if rank == 0 else [theirs, mine])[:numel]
    assert torch.equal(joined, ref["flat"][:numel])


def test_c3_sh48_properties_and_masked_parity(gs, cuda):
    """C3 (2.4 M Gaussians, 1080p) at D = 48: the per-Gaussian frame is bit-deterministic, launches as many of our
    kernels as the RGB frame, bins the same M and consumes the same M_eff as the RGB frame on the same geometry, and
    matches the fp64 oracle on sampled tiles (upstream gradient non-zero only there; every other gradient exactly 0)."""
    import renderer
    n, w, h = 2_400_000, 1920, 1080
    g48 = S.make_gaussians(n, w, h, 0, sh_dim=48)
    g3 = S.make_gaussians(n, w, h, 0, sh_dim=3)          # the generator draws colours last: the same geometry
    v = S.make_view(w, h, 0)
    cam = O.Camera(w, h, v.fx, v.fy, v.rot, v.tran, v.near)
    go = (torch.rand(h, w, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1).to(cuda)

    def frame(rctx, gg):
        d = {q: t.clone().requires_grad_(True) for q, t in gg.items()}
        l0 = gs[0].kernel_launches()
        img, _ = renderer.render_frame_final(rctx, *(d[q] for q in NAMES), *_args(v))
        img.backward(go)
        torch.cuda.synchronize()
        st = rctx.stats()
        return [img.detach()] + [d[q].grad for q in NAMES], gs[0].kernel_launches() - l0, st

    dev48 = {q: t.to(cuda) for q, t in g48.items()}
    dev3 = {q: t.to(cuda) for q, t in g3.items()}
    rctx = _ctx(gs, "gaussian")
    frame(rctx, dev48)                                     # the first frame of a context also fills its index table
    a, la, sa = frame(rctx, dev48)
    b, lb, sb = frame(rctx, dev48)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    del a, b
    r3 = _ctx(gs, "gaussian")                              # d = 3 ignores the setting
    frame(r3, dev3)
    _, l3, s3 = frame(r3, dev3)
    assert la == lb == l3
    assert (sa["n_instances"], sa["n_instances_eff"]) == (s3["n_instances"], s3["n_instances_eff"])
    del dev3, r3

    # masked-gradient parity on sampled tiles (the style of test_scale_parity_gpu.py)
    sp = _splatter(g48, v, cuda, sh_eval="gaussian")
    with torch.no_grad():
        sp(0)
    idx, accum = sp._rctx.sorted_instances()
    idx, accum = idx.cpu(), accum.cpu().long()
    neff = sp._rctx.tile_consumed().cpu().long()
    tiles = _pick_tiles(accum, neff, cam.ntx, cam.nty, 5)
    assert int((accum[1:] - accum[:-1]).max()) > 1000     # multi-chunk tiles really are exercised
    top, left = (cam.Hp - h) // 2, (cam.Wp - w) // 2
    gom = S.make_grad_output(h, w, 0) * (h * w) * _tile_mask(cam, tiles, h, w)
    img = sp(0)
    img.backward(gom.to(cuda))
    opad, U, ograds = _oracle_on_tiles(g48, cam, idx, accum, tiles, gom)
    raw = torch.zeros(cam.Hp, cam.Wp, 3, dtype=torch.float64)
    raw[top:top + h, left:left + w] = img.detach().cpu().double()
    for t in tiles:
        ty, tx = divmod(t, cam.ntx)
        r0, r1 = max(ty * 16, top), min((ty + 1) * 16, top + h)
        assert abs_err(raw[r0:r1, tx * 16:(tx + 1) * 16], opad[r0:r1, tx * 16:(tx + 1) * 16].clamp(0, 1)) < IMG_ATOL, t
    other = torch.ones(n, dtype=torch.bool)
    other[U] = False
    for q in NAMES:
        got = getattr(sp.gaussian_3ds, q).grad.cpu()
        assert bool(torch.isfinite(got).all()), q
        assert rel_err(got[U], ograds[q]) < GRAD_RTOL, q
        assert float(got[other].abs().max()) == 0.0, q


def _oracle_on_tiles(g, cam, idx, accum, tiles, go_final):
    """fp64 per-Gaussian SH oracle restricted to the Gaussians the DEVICE binned into `tiles`, in the device's order
    (binning and order parity are checked elsewhere).  Returns (padded image, U, gradients on U)."""
    dt = torch.float64
    ids = [idx[int(accum[t]):int(accum[t + 1])].long() for t in tiles]
    U = torch.unique(torch.cat(ids))
    p = {k: g[k][U].to(dt).clone().requires_grad_(True) for k in NAMES}
    logits = G.gaussian_logits(p["pos"], p["rgb"], cam)
    nq, ns, opa_a, rgb_a = O.preactivate(p["quat"], p["scale"], p["opa"], logits)
    rp, rc, _ = O.global_culling(p["pos"], nq, ns, cam.rot.to(dt), cam.tran.to(dt), cam.near, cam.half_w, cam.half_h)
    loc = torch.cat([torch.searchsorted(U, i) for i in ids])
    counts = torch.zeros(cam.ntx * cam.nty, dtype=torch.int64)
    for t, i in zip(tiles, ids):
        counts[t] = i.numel()
    acc2 = torch.zeros(cam.ntx * cam.nty + 1, dtype=torch.int64)
    acc2[1:] = torch.cumsum(counts, 0)
    padded = O.draw(rp[loc], rgb_a[loc], opa_a[loc], rc[loc], acc2.to(torch.int32), cam.Hp, cam.Wp, cam.fx, cam.fy,
                    tiles=torch.tensor(tiles))
    cam.crop(torch.clamp(padded, 0, 1)).backward(go_final.to(dt))
    return padded.detach(), U, {k: p[k].grad for k in NAMES}
