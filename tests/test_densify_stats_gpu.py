"""Screen-space densification statistics on the fused frame path (gs_ctx_set_densify_stats,
RenderContext.set_densify_stats, `Splatter(..., densify_stats=...)`) against the fp64 oracle of
tests/densify_stats_oracle.py, accumulated over 3 views; their lifetime and error rules; and densification from them
(`Splatter.adaptive_control_screen`) against the scored oracle plan."""
import ctypes
import math
import os

import pytest
import torch

import densify_stats_oracle as DS
import gs_oracle as O
import sh_gaussian_oracle as G
import synthetic as S
from helpers import device_depth_keys
from test_scale_parity_gpu import _pick_tiles, _tile_mask

pytestmark = pytest.mark.gpu

NAMES = ("pos", "rgb", "opa", "quat", "scale")
STAT_RTOL = 1e-3
# case: (colour width, sh_eval, filter2d, maps, packed, absgrad)
CASES = {
    "rgb": (3, "pixel", "none", False, False, True),
    "sh27-gauss": (27, "gaussian", "none", False, False, True),
    "sh48-gauss": (48, "gaussian", "none", False, False, True),
    "sh27-pixel": (27, "pixel", "none", False, False, False),
    "rgb-maps": (3, "pixel", "none", True, False, True),
    "sh27-gauss-maps": (27, "gaussian", "none", True, False, True),
    "rgb-dilate": (3, "pixel", "dilate", False, False, True),
    "rgb-antialias": (3, "pixel", "antialias", False, False, True),
    "rgb-packed": (3, "pixel", "none", False, True, False),
}


def _views(w, h, k=3):
    return [S.make_view(w, h, j) for j in range(k)]


def _vdict(v):
    return dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)


def _cam(v):
    return O.Camera(v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near)


def _splatter(g, views, dev, **kw):
    import splatter
    return splatter.Splatter.from_tensors(g, [_vdict(v) for v in views], device=dev,
                                          use_sh_coeff=g["rgb"].shape[1] != 3, **kw)


def _upstream(shape, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(shape, generator=gen, dtype=torch.float64) * 2 - 1


def _device_frame(sp, v, j, final, maps, seed):
    """One forward + backward of view j (v) with a seeded upstream gradient; returns the oracle's loss function."""
    cam = _cam(v)
    if maps:
        o = sp.render_maps(j)
        gi, gd, ga = (_upstream(o[k].shape, seed + i) for i, k in enumerate(("image", "depth", "alpha")))
        dev = o["image"].device
        L = (o["image"] * gi.float().to(dev)).sum() + (o["depth"] * gd.float().to(dev)).sum() + \
            (o["alpha"] * ga.float().to(dev)).sum()
        L.backward()

        def loss(out):
            return ((cam.crop(torch.clamp(out["padded"], 0, 1)) * gi).sum() +
                    (cam.crop(out["depth"].unsqueeze(-1)).squeeze(-1) * gd).sum() +
                    (cam.crop(out["alpha"].unsqueeze(-1)).squeeze(-1) * ga).sum())
        return loss
    if final:
        img = sp(j)
        go = _upstream(img.shape, seed)
        img.backward(go.float().to(img.device))
        return lambda out: (cam.crop(torch.clamp(out["padded"], 0, 1)) * go).sum()
    sp.set_camera(j)
    img = sp.render_padded()
    go = _upstream(img.shape, seed)
    img.backward(go.float().to(img.device))
    return lambda out: (out["padded"] * go).sum()


def _oracle_stats(g, views, losses, sh_eval, mode, maps, absgrad, dev):
    p = {q: t.double() for q, t in g.items()}
    n = p["pos"].shape[0]
    acc = dict(grad2d=torch.zeros(n, dtype=torch.float64), absgrad=torch.zeros(n, dtype=torch.float64),
               count=torch.zeros(n, dtype=torch.int64), radius=torch.zeros(n, dtype=torch.float64))
    for v, loss in zip(views, losses):
        cam = _cam(v)
        rgb, use_sh = p["rgb"], False
        if p["rgb"].shape[1] != 3:
            if sh_eval == "gaussian":
                rgb = G.gaussian_logits(p["pos"], p["rgb"], cam)
            else:
                use_sh = True
        r = DS.frame_stats(p["pos"], rgb, p["opa"], p["quat"], p["scale"], cam, loss, mode=mode, use_sh_coeff=use_sh,
                           maps=maps, absgrad=absgrad, depth_key=device_depth_keys(g, cam, dev))
        acc["grad2d"] += r["grad2d"]
        acc["count"] += r["count"]
        acc["radius"] = torch.maximum(acc["radius"], r["radius"])
        if absgrad:
            acc["absgrad"] += r["absgrad"]
    return acc


def _check(st, ref, absgrad):
    for k in ("grad2d",) + (("absgrad",) if absgrad else ()):
        got = getattr(st, k).double().cpu()
        scale = float(ref[k].abs().max())
        assert scale > 0, k
        assert float((got - ref[k]).abs().max()) < STAT_RTOL * scale, (k, float((got - ref[k]).abs().max()), scale)
    assert torch.equal(st.count.cpu().long(), ref["count"])
    got_r = st.max_radius.double().cpu()
    want_r = torch.ceil(ref["radius"])
    frac = ref["radius"] - torch.floor(ref["radius"])
    near_int = (frac < 1e-4) | (frac > 1 - 1e-4)
    bad = (got_r != want_r) & ~near_int
    assert not bool(bad.any()), (got_r[bad][:5], ref["radius"][bad][:5])


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("case", list(CASES))
def test_stats_vs_oracle(gs, cuda, case, final):
    """grad2d / absgrad within 1e-3 of the largest reference value, count exact, max_radius exact (except where the
    oracle's radius is within 1e-4 of an integer), over 3 views."""
    sh_dim, sh_eval, mode, maps, packed, absgrad = CASES[case]
    if maps and not final:
        pytest.skip("the maps are checked through Splatter.render_maps (final)")
    n, w, h = (4000, 128, 96) if sh_dim == 3 or sh_eval == "gaussian" else (2500, 112, 80)
    g = S.make_gaussians(n, w, h, 0, sh_dim, (0.05, 0.9), (0.6, 5.0))
    views = _views(w, h)
    if packed:
        gs[0].tune("gather", 0)
    try:
        sp = _splatter(g, views, cuda, sh_eval=sh_eval, filter2d=mode,
                       densify_stats="absgrad" if absgrad else "grad")
        losses = [_device_frame(sp, v, j, final, maps, 10 * j) for j, v in enumerate(views)]
        torch.cuda.synchronize()
    finally:
        gs[0].tune("gather", 1)
    ref = _oracle_stats(g, views, losses, sh_eval, mode, maps, absgrad, cuda)
    _check(sp.densify_stats, ref, absgrad)


def _grads(sp):
    return [getattr(sp.gaussian_3ds, q).grad.clone() for q in NAMES]


@pytest.mark.parametrize("sh_dim,sh_eval", [(3, "pixel"), (48, "gaussian")])
def test_gradients_bit_identical_and_stats_deterministic(gs, cuda, sh_dim, sh_eval):
    """Image and parameter gradients are the same bits with statistics off, grad and absgrad; two runs give the same
    statistics bit for bit."""
    g = S.make_gaussians(6000, 192, 128, 1, sh_dim, (0.05, 0.9), (0.6, 5.0))
    views = _views(192, 128)
    go = [_upstream((128, 192, 3), j).float().to(cuda) for j in range(3)]
    outs = {}
    for mode in ("none", "grad", "absgrad", "absgrad2"):
        sp = _splatter(g, views, cuda, sh_eval=sh_eval, densify_stats=mode.rstrip("2"))
        imgs, grads = [], []
        for j in range(3):
            img = sp(j)
            img.backward(go[j])
            imgs.append(img.detach().clone())
            grads.append(_grads(sp))
            for q in NAMES:
                getattr(sp.gaussian_3ds, q).grad = None
        torch.cuda.synchronize()
        outs[mode] = (imgs, grads, sp.densify_stats)
    for mode in ("grad", "absgrad"):
        for a, b in zip(outs["none"][0], outs[mode][0]):
            assert torch.equal(a, b), mode
        for ga, gb in zip(outs["none"][1], outs[mode][1]):
            for x, y in zip(ga, gb):
                assert torch.equal(x, y), mode
    s1, s2 = outs["absgrad"][2], outs["absgrad2"][2]
    for k in ("grad2d", "absgrad", "count", "max_radius"):
        assert torch.equal(getattr(s1, k), getattr(s2, k)), k
    assert torch.equal(outs["grad"][2].grad2d, s1.grad2d)
    assert int(s1.count.max()) == 3 and float(s1.absgrad.sum()) > float(s1.grad2d.sum())


def test_every_backward_variant_accumulates_but_camera_only(gs, cuda):
    """final (Splatter.forward), aux (render_maps) and cam with parameter gradients (render_at_pose) accumulate; a
    camera-only backward (no parameter needs a gradient) leaves the statistics alone."""
    g = S.make_gaussians(3000, 128, 96, 2, 3, (0.05, 0.9), (0.6, 5.0))
    views = _views(128, 96, 1)
    sp = _splatter(g, views, cuda, densify_stats="absgrad")
    st = sp.densify_stats
    snap = lambda: [t.clone() for t in (st.grad2d, st.absgrad, st.count, st.max_radius)]
    sp(0).sum().backward()
    a = snap()
    assert int(a[2].max()) == 1 and float(a[0].sum()) > 0 and float(a[1].sum()) > 0
    o = sp.render_maps(0)
    (o["image"].sum() + o["depth"].sum()).backward()
    b = snap()
    assert int(b[2].max()) == 2 and float(b[0].sum()) > float(a[0].sum())
    rot = views[0].rot.float().to(cuda).requires_grad_(True)
    tran = views[0].tran.float().to(cuda).requires_grad_(True)
    sp.render_at_pose(rot, tran, camera_id=0)["image"].sum().backward()
    c = snap()
    assert int(c[2].max()) == 3 and float(c[0].sum()) > float(b[0].sum())
    for q in NAMES:
        getattr(sp.gaussian_3ds, q).requires_grad_(False)
    sp.render_at_pose(rot, tran, camera_id=0)["image"].sum().backward()
    torch.cuda.synchronize()
    assert rot.grad is not None
    for x, y in zip(c, snap()):
        assert torch.equal(x, y)


def _raw(gs, g, v, cuda, sh_eval="pixel"):
    import renderer
    rctx = gs[0].RenderContext()
    rctx.set_sh_eval(renderer.SH_EVAL[sh_eval])
    p = {q: t.to(cuda) for q, t in g.items()}
    img, _ = rctx.forward(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], v.width, v.height, v.fx, v.fy, v.rot,
                          v.tran, v.near, 0.05, 0)
    return rctx, p, img


def _stats(n, cuda, absgrad=False):
    z = lambda dt=torch.float32: torch.zeros(n, device=cuda, dtype=dt)
    return dict(grad2d=z(), count=z(torch.int32), max_radius=z(), absgrad=z() if absgrad else None)


def _backward_into(rctx, p, img, outs=None):
    outs = [torch.full_like(p[q], float("nan")) for q in NAMES] if outs is None else outs
    rctx.backward_into(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], img, torch.ones_like(img), *outs)
    return outs


# case: (colour width, knob set for the whole test, knob set for the backward only, its shipped value)
REFUSALS = {"n-mismatch": (3, None, None), "absgrad-sh-pixel": (27, None, None),
            "absgrad-packed": (3, ("gather", 0, 1), None), "absgrad-knobs": (3, None, ("bwd_unroll", 2, 4))}


@pytest.mark.parametrize("case", list(REFUSALS))
def test_refusals_before_any_launch(gs, cuda, case):
    """An n mismatch, and absgrad on a per-pixel SH frame, on the packed path or with non-default backward blend knobs,
    fail before any launch: the gradient buffers stay unwritten and the statistics untouched."""
    sh_dim, knob_all, knob_bwd = REFUSALS[case]
    g = S.make_gaussians(2000, 96, 64, 3, sh_dim, (0.05, 0.9), (0.6, 5.0))
    v = S.make_view(96, 64, 0)
    if knob_all:
        gs[0].tune(knob_all[0], knob_all[1])
    try:
        rctx, p, img = _raw(gs, g, v, cuda)
        s = _stats(2001 if case == "n-mismatch" else 2000, cuda, absgrad=case != "n-mismatch")
        rctx.set_densify_stats(**s)
        if knob_bwd:
            gs[0].tune(knob_bwd[0], knob_bwd[1])
        outs = [torch.full_like(p[q], float("nan")) for q in NAMES]
        torch.cuda.synchronize()
        before = gs[0].kernel_launches()
        with pytest.raises(RuntimeError, match="densify statistics|sized for another n"):
            _backward_into(rctx, p, img, outs)
        torch.cuda.synchronize()
        assert gs[0].kernel_launches() == before
    finally:
        for k in (knob_all, knob_bwd):
            if k:
                gs[0].tune(k[0], k[2])
    for o in outs:
        assert bool(torch.isnan(o).all())
    assert float(s["grad2d"].abs().sum()) == 0 and int(s["count"].sum()) == 0
    rctx.clear_densify_stats()
    outs = _backward_into(rctx, p, img)      # cleared: the backward runs
    assert bool(torch.isfinite(outs[0]).all())


def test_stats_launch_count(gs, cuda):
    """The statistics add exactly one launch to a backward."""
    g = S.make_gaussians(2000, 96, 64, 4, 3, (0.05, 0.9), (0.6, 5.0))
    v = S.make_view(96, 64, 0)
    rctx, p, img = _raw(gs, g, v, cuda)
    b0 = gs[0].kernel_launches()
    _backward_into(rctx, p, img)
    plain = gs[0].kernel_launches() - b0
    rctx.set_densify_stats(**_stats(2000, cuda, absgrad=True))
    img, _ = rctx.forward(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], v.width, v.height, v.fx, v.fy, v.rot,
                          v.tran, v.near, 0.05, 0)
    b1 = gs[0].kernel_launches()
    _backward_into(rctx, p, img)
    assert gs[0].kernel_launches() - b1 == plain + 1


def test_adaptive_control_screen_vs_oracle(gs, cuda):
    """Splatter.adaptive_control_screen against the scored oracle plan with the same generator: same counts, same
    layout, parameters within 1e-6; the statistics restart at the new n."""
    g = S.make_gaussians(3000, 128, 96, 5, 3, (0.05, 0.9), (0.6, 5.0))
    views = _views(128, 96)
    sp = _splatter(g, views, cuda, densify_stats="absgrad")
    for j in range(3):
        img = sp(j)
        img.backward(_upstream(img.shape, j).float().to(cuda))
    st = sp.densify_stats
    accum, count, rad = st.absgrad.double().cpu(), st.count.cpu(), st.max_radius.double().cpu()
    thr = float((accum / count.clamp(min=1)).quantile(0.8))
    norm = sp.gaussian_3ds.scale.detach().norm(dim=-1)
    tau = float(norm.median())
    before = {q: getattr(sp.gaussian_3ds, q).detach().double().cpu() for q in NAMES}
    gen = torch.Generator(device=cuda).manual_seed(11)
    info = sp.adaptive_control_screen(tau, 10.0, grad_thresh=thr, use_abs=True, max_screen_size=20, generator=gen)
    n_split = info["split"]
    z = torch.randn(2, n_split, 3, generator=torch.Generator(device=cuda).manual_seed(11), device=cuda).double().cpu()
    ref, rinfo = DS.adaptive_control_stats(*(before[q] for q in NAMES), accum, count, tau, 10.0, grad_thresh=thr,
                                           max_radius=rad, max_screen_px=20.0, z=z)
    assert info["cloned"] > 0 and info["split"] > 0
    assert (info["deleted"], info["cloned"], info["split"]) == (rinfo["deleted"], rinfo["cloned"], rinfo["split"])
    for q, r in zip(NAMES, ref):
        got = getattr(sp.gaussian_3ds, q).detach().double().cpu()
        assert got.shape == r.shape, q
        assert float((got - r).abs().max()) < 1e-6 * max(1.0, float(r.abs().max())), q
    assert st.n == info["total"] and int(st.count.sum()) == 0


def test_short_3dgs_loop_densifies_twice(gs, cuda):
    """A 3DGS-style loop (absgrad statistics, dilation, per-Gaussian SH) on synthetic views: Adam steps, two
    densifications, the statistics follow the scene."""
    n, w, h = 3000, 128, 96
    g = S.make_gaussians(n, w, h, 6, 27, (0.05, 0.9), (0.6, 5.0))
    views = _views(w, h, 4)
    tgt = [S.make_grad_output(h, w, j).to(cuda).abs() * (h * w) for j in range(4)]
    sp = _splatter(g, views, cuda, sh_eval="gaussian", filter2d="dilate", densify_stats="absgrad")
    totals = []
    for rnd in range(2):
        opt = torch.optim.Adam(sp.gaussian_3ds.parameters(), lr=1e-3)
        for it in range(8):
            j = it % 4
            loss = (sp(j) - tgt[j]).abs().mean()
            opt.zero_grad()
            loss.backward()
            opt.step()
        assert int(sp.densify_stats.count.max()) >= 2
        info = sp.adaptive_control_screen(0.01, 10.0, grad_thresh=1e-7, use_abs=True, max_screen_size=200)
        totals.append(info["total"])
        assert info["total"] == sp.gaussian_3ds.pos.shape[0] == sp.densify_stats.n
    torch.cuda.synchronize()
    assert totals[0] != n and math.isfinite(float(loss))


class _Stats(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int), ("grad2d", ctypes.c_void_p), ("absgrad", ctypes.c_void_p),
                ("count", ctypes.c_void_p), ("max_radius", ctypes.c_void_p)]


def _lib():
    pkg = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "3d-gaussian-splatting_b200")
    lib = ctypes.CDLL(os.path.join(pkg, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_ctx_set_densify_stats.argtypes = [ctypes.c_void_p, ctypes.POINTER(_Stats)]
    lib.gs_ctx_destroy.argtypes = [ctypes.c_void_p]
    return lib


def test_host_entry_point_accumulates_and_setter_checks(gs, cuda):
    """gs_render_forward_backward_host accumulates the same statistics, bit for bit, as the Python path of the same
    padded frame; gs_ctx_set_densify_stats on a real context refuses n < 0 and a NULL grad2d / count / max_radius with
    n > 0, takes a NULL absgrad, and NULL turns the statistics off."""
    n, w, h = 3000, 112, 80
    g = S.make_gaussians(n, w, h, 0, 3, (0.05, 0.9), (0.6, 5.0))
    v = S.make_view(w, h, 1)
    cam = _cam(v)
    gpad = torch.zeros(cam.Hp, cam.Wp, 3)
    gpad[:h, :w] = S.make_grad_output(h, w, 0) * (h * w)
    sp = _splatter(g, [v], cuda, densify_stats="absgrad")
    sp.set_camera(0)
    sp.render_padded().backward(gpad.to(cuda))
    want = sp.densify_stats

    lib = _lib()

    class Cam(ctypes.Structure):
        _fields_ = [("width", ctypes.c_int), ("height", ctypes.c_int), ("focal_x", ctypes.c_float),
                    ("focal_y", ctypes.c_float), ("rot", ctypes.c_float * 9), ("tran", ctypes.c_float * 3),
                    ("near_plane", ctypes.c_float), ("tile_thresh", ctypes.c_float)]
    P = ctypes.c_void_p
    ctx = P()
    assert lib.gs_ctx_create(ctypes.byref(ctx)) == 0
    try:
        st = _stats(n, cuda, absgrad=True)
        ptr = {k: (t.data_ptr() if t is not None else None) for k, t in st.items()}
        for bad in (_Stats(-1, ptr["grad2d"], None, ptr["count"], ptr["max_radius"]),
                    _Stats(n, None, None, ptr["count"], ptr["max_radius"]),
                    _Stats(n, ptr["grad2d"], None, None, ptr["max_radius"]),
                    _Stats(n, ptr["grad2d"], None, ptr["count"], None)):
            assert lib.gs_ctx_set_densify_stats(ctx, ctypes.byref(bad)) == -1
            assert b"gs_ctx_set_densify_stats" in lib.gs_last_error()
        assert lib.gs_ctx_set_densify_stats(ctx, ctypes.byref(_Stats(n, ptr["grad2d"], None, ptr["count"],
                                                                     ptr["max_radius"]))) == 0
        assert lib.gs_ctx_set_densify_stats(ctx, None) == 0
        assert lib.gs_ctx_set_densify_stats(ctx, ctypes.byref(_Stats(n, ptr["grad2d"], ptr["absgrad"], ptr["count"],
                                                                     ptr["max_radius"]))) == 0
        c = Cam(w, h, v.fx, v.fy, (ctypes.c_float * 9)(*v.rot.flatten().tolist()),
                (ctypes.c_float * 3)(*v.tran.tolist()), 0.3, 0.05)
        dev = {k: t.to(cuda).contiguous() for k, t in g.items()}
        grads = {k: torch.empty_like(t) for k, t in dev.items()}
        gimg_host = gpad.contiguous().pin_memory()
        img_host = torch.empty(cam.Hp, cam.Wp, 3).pin_memory()
        lib.gs_render_forward_backward_host.argtypes = [P] * 6 + [ctypes.c_int] * 3 + [ctypes.POINTER(Cam)] + [P] * 8
        torch.cuda.synchronize()
        rc = lib.gs_render_forward_backward_host(
            ctx, *(dev[k].data_ptr() for k in NAMES), n, 3, 0, ctypes.byref(c), gimg_host.data_ptr(),
            img_host.data_ptr(), *(grads[k].data_ptr() for k in NAMES), None)
        assert rc == 0, lib.gs_last_error()
        torch.cuda.synchronize()
    finally:
        lib.gs_ctx_destroy(ctx)
    assert int(st["count"].sum()) > 0 and float(st["absgrad"].sum()) > 0
    for k in ("grad2d", "absgrad", "count", "max_radius"):
        assert torch.equal(st[k], getattr(want, k)), k


@pytest.mark.parametrize("rank", [0, 1])
def test_push_on_one_gpu_accumulates(gs, cuda, rank):
    """With the data-parallel push (world = 2, both staging buffers on this device) the backward accumulates the same
    statistics, bit for bit, as without it."""
    import renderer
    n, w, h = 4000, 128, 96
    g = S.make_gaussians(n, w, h, 0, 3, (0.05, 0.9), (0.6, 5.0))
    v = S.make_view(w, h, 1)
    go = _upstream((h, w, 3), 0).float().to(cuda)
    world = 2

    def run(push):
        def alloc(numel, device):
            per = (numel + world * 4 - 1) // (world * 4) * 4
            flat = torch.zeros(world * per, device=device)
            if not push:
                return flat
            staging = [torch.zeros(world * per, device=device) for _ in range(world)]
            alloc.keep = staging
            return flat, (flat.data_ptr(), [t.data_ptr() for t in staging], per, rank)

        rctx = gs[0].RenderContext()
        st = _stats(n, cuda, absgrad=True)
        rctx.set_densify_stats(**st)
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        renderer.set_flat_grad_allocator(alloc)
        try:
            img, _ = renderer.render_frame_final(rctx, *(d[q] for q in NAMES), v.width, v.height, v.fx, v.fy, v.rot,
                                                 v.tran, v.near, 0.05, "abs")
            img.backward(go)
        finally:
            renderer.set_flat_grad_allocator(None)
        torch.cuda.synchronize()
        return st

    ref, got = run(False), run(True)
    assert int(ref["count"].sum()) > 0 and float(ref["absgrad"].sum()) > 0
    for k in ("grad2d", "absgrad", "count", "max_radius"):
        assert torch.equal(got[k], ref[k]), k


def test_c3_masked_tiles_vs_oracle(gs, cuda):
    """C3 (2.4 M Gaussians, 1080p, RGB, absgrad): with the upstream gradient non-zero only on sampled tiles, the
    statistics of the Gaussians the device binned there match the fp64 oracle, and every other Gaussian's grad2d and
    absgrad are exactly 0."""
    n, w, h = 2_400_000, 1920, 1080
    g = S.make_gaussians(n, w, h, 0)
    v = S.make_view(w, h, 0)
    cam = _cam(v)
    sp = _splatter(g, [v], cuda, densify_stats="absgrad")
    with torch.no_grad():
        sp(0)
    idx, accum = sp._rctx.sorted_instances()
    idx, accum = idx.cpu(), accum.cpu().long()
    neff = sp._rctx.tile_consumed().cpu().long()
    tiles = _pick_tiles(accum, neff, cam.ntx, cam.nty, 5)
    gom = (S.make_grad_output(h, w, 0) * (h * w) * _tile_mask(cam, tiles, h, w)).double()
    sp(0).backward(gom.float().to(cuda))
    torch.cuda.synchronize()
    st = sp.densify_stats
    ids = [idx[int(accum[t]):int(accum[t + 1])].long() for t in tiles]
    U, ref = DS.tile_stats(g["pos"], g["rgb"], g["opa"], g["quat"], g["scale"], cam, ids, tiles,
                           lambda out: (cam.crop(torch.clamp(out["padded"], 0, 1)) * gom).sum())
    for k in ("grad2d", "absgrad"):
        got = getattr(st, k).double().cpu()
        scale = float(ref[k].abs().max())
        assert scale > 0, k
        assert float((got[U] - ref[k]).abs().max()) < STAT_RTOL * scale, (k, float((got[U] - ref[k]).abs().max()))
        other = torch.ones(n, dtype=torch.bool)
        other[U] = False
        assert float(got[other].abs().max()) == 0.0, k
    assert bool((st.count.cpu()[U] == 1).all())
    got_r, rr = st.max_radius.double().cpu()[U], ref["radius"]
    frac = rr - torch.floor(rr)
    bad = (got_r != torch.ceil(rr)) & ~((frac < 1e-4) | (frac > 1 - 1e-4))
    assert not bool(bad.any()), (got_r[bad][:5], rr[bad][:5])
