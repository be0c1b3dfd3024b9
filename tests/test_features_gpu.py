"""Feature maps on the fused frame path (renderer.render_frame_feat, gs_render_forward_feat / gs_render_backward_feat)
against the fp64 oracle of tests/feat_oracle.py, bit-identity with the aux frame, determinism, the refusals, and the
features following densification."""
import pytest
import torch

import feat_oracle as FT
import synthetic as S
from helpers import abs_err, device_depth_keys, rel_err, scene

pytestmark = pytest.mark.gpu

GRAD_RTOL = 1e-3
BG = (0.2, 0.5, 0.9)
NAMES = ("pos", "rgb", "opa", "quat", "scale")


def _args(v):
    return (v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")


def _feat(n, F, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(n, F, generator=gen) * 4 - 2


def _ctx(gs, sh_gaussian=False, filter2d="none"):
    import renderer
    rctx = gs[0].RenderContext()
    rctx.set_sh_eval(renderer.SH_EVAL["gaussian" if sh_gaussian else "pixel"])
    rctx.set_filter2d(renderer.FILTER2D[filter2d], 0.3)
    return rctx


CASES = [  # (F, sh_dim, filter2d, maps + background)
    (8, 3, "none", True),
    (16, 3, "none", False),
    (32, 3, "none", True),
    (16, 27, "none", True),
    (8, 48, "none", False),
    (32, 48, "none", True),
    (16, 3, "antialias", True),
]


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("F,sh_dim,filter2d,maps", CASES)
def test_feat_frame_vs_oracle(gs, cuda, F, sh_dim, filter2d, maps, final):
    import renderer
    n = 3000
    g, v, cam = scene(n, 112, 80, k=1, sh_dim=sh_dim, opa_range=(0.05, 0.9))
    feat = _feat(n, F, 3)
    sh = sh_dim != 3
    bg = BG if maps else None
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    pf = feat.double().clone().requires_grad_(True)
    o = FT.render_feat(*(p[q] for q in NAMES), pf, cam, mode=filter2d, background=bg, sh_gaussian=sh,
                       depth_key=device_depth_keys(g, cam, cuda))
    pre = "" if final else "padded_"
    oi, of, od, oa = (o[pre + k] for k in ("image", "features", "depth", "alpha"))
    rctx = _ctx(gs, sh, filter2d)
    gen = torch.Generator().manual_seed(5)
    gi = (torch.rand(*oi.shape, generator=gen) * 2 - 1).double()
    gf = (torch.rand(*of.shape, generator=gen) * 2 - 1).double()
    gd = (torch.rand(*od.shape, generator=gen) * 2 - 1).double() if maps else None
    ga = (torch.rand(*oa.shape, generator=gen) * 2 - 1).double() if maps else None
    cases = {"features": (None, gf), "image": (gi, None), "mixed": (gi, gf)}
    for case, (ugi, ugf) in cases.items():
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        df = feat.to(cuda).clone().requires_grad_(True)
        img, fm, dep, alp, _ = renderer.render_frame_feat(rctx, *(d[q] for q in NAMES), df, *_args(v), background=bg,
                                                          final=final)
        assert abs_err(img, oi) < 1e-4
        assert abs_err(fm, of) < 1e-4 * max(1.0, float(feat.abs().max()))
        assert abs_err(alp, oa) < 1e-4
        mixed = case == "mixed"
        trip = [(m, t, u) for m, t, u in ((img, oi, ugi), (fm, of, ugf), (dep, od, gd if mixed else None),
                                          (alp, oa, ga if mixed else None)) if u is not None]
        ref = torch.autograd.grad([t for _, t, _ in trip], [p[q] for q in NAMES] + [pf], [u for _, _, u in trip],
                                  retain_graph=True, allow_unused=True)
        torch.autograd.backward([m for m, _, _ in trip], [u.float().to(cuda) for _, _, u in trip])
        for q, r, mine in zip(NAMES + ("feat",), ref, [d[q].grad for q in NAMES] + [df.grad]):
            r = torch.zeros_like(mine, dtype=torch.float64, device="cpu") if r is None else r
            assert rel_err(mine, r) < GRAD_RTOL, (case, q, rel_err(mine, r))


@pytest.mark.parametrize("F", [8, 16, 32])
def test_feat_frame_matches_aux_frame(gs, cuda, F):
    """Image, depth and alpha are bit-identical to the aux frame's; with the features unused the parameter gradients
    are too and grad_feat is zero; an explicit zero feature gradient runs the feature kernels and agrees closely.
    Two feature backwards are bit-equal."""
    import renderer
    n = 10000
    g, v, _ = scene(n, 256, 256, opa_range=(0.05, 0.9))
    feat = _feat(n, F, 1).to(cuda)
    gen = torch.Generator().manual_seed(2)
    gi = (torch.rand(256, 256, 3, generator=gen) * 2 - 1).to(cuda)
    gd = (torch.rand(256, 256, generator=gen) * 2 - 1).to(cuda)
    gf = (torch.rand(256, 256, F, generator=gen) * 2 - 1).to(cuda)
    rctx = gs[0].RenderContext()
    res = {}
    for mode in ("aux", "unused", "zero", "grad", "grad2"):
        d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
        df = feat.clone().requires_grad_(True)
        if mode == "aux":
            img, dep, alp, _ = renderer.render_frame_aux(rctx, *(d[q] for q in NAMES), *_args(v), background=BG)
            torch.autograd.backward([img, dep], [gi, gd])
            fm = None
        else:
            img, fm, dep, alp, _ = renderer.render_frame_feat(rctx, *(d[q] for q in NAMES), df, *_args(v),
                                                              background=BG)
            up = {"unused": None, "zero": torch.zeros_like(gf), "grad": gf, "grad2": gf}[mode]
            torch.autograd.backward([img, dep] + ([fm] if up is not None else []), [gi, gd] + ([up] if up is not None
                                                                                                 else []))
        torch.cuda.synchronize()
        res[mode] = dict(out=[img.detach(), dep.detach(), alp.detach()], grads=[d[q].grad for q in NAMES],
                         gfeat=None if fm is None else df.grad, fm=None if fm is None else fm.detach())
    for mode in ("unused", "zero", "grad"):
        for a, b in zip(res[mode]["out"], res["aux"]["out"]):
            assert torch.equal(a, b), mode
    for a, b in zip(res["unused"]["grads"], res["aux"]["grads"]):
        assert torch.equal(a, b)
    assert torch.equal(res["unused"]["gfeat"], torch.zeros_like(feat))
    assert torch.equal(res["zero"]["gfeat"], torch.zeros_like(feat))
    # the feature backward sums the same per-(pixel, instance) terms in another order than the shipped RGB kernel
    # (reduce8 over warps of 2-pixel threads, not 8-pixel rows), so fp32 reassociation is all that differs
    for q, a, b in zip(NAMES, res["zero"]["grads"], res["aux"]["grads"]):
        assert rel_err(a, b) < 1e-5, q
    assert float(res["grad"]["gfeat"].abs().max()) > 0
    for a, b in zip(res["grad"]["grads"] + [res["grad"]["gfeat"], res["grad"]["fm"]],
                    res["grad2"]["grads"] + [res["grad2"]["gfeat"], res["grad2"]["fm"]]):
        assert torch.equal(a, b)


def _raises_before_launch(gs, fn, match):
    torch.cuda.synchronize()
    l0 = gs[0].kernel_launches()
    with pytest.raises(RuntimeError, match=match):
        fn()
    assert gs[0].kernel_launches() == l0


def test_feat_refusals(gs, cuda):
    n, F = 2000, 16
    g, v, _ = scene(n, 96, 64)
    g27, _, _ = scene(n, 96, 64, sh_dim=27)
    d = {q: t.to(cuda).contiguous() for q, t in g.items()}
    d27 = {q: t.to(cuda).contiguous() for q, t in g27.items()}
    feat = _feat(n, F, 0).to(cuda)
    rctx = gs[0].RenderContext()
    cam = (v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, 0)

    def fwd(p, f, **kw):
        return rctx.forward_feat(*(p[q] for q in NAMES), f, *cam, **kw)

    _raises_before_launch(gs, lambda: fwd(d27, feat), "per pixel")
    _raises_before_launch(gs, lambda: fwd(d, _feat(n, 12, 0).to(cuda)), "8, 16 or 32")
    mis = torch.empty(n * F + 1, device=cuda)[1:].view(n, F)
    mis.copy_(feat)
    _raises_before_launch(gs, lambda: fwd(d, mis), "aligned")
    gs[0].tune("gather", 0)
    try:
        _raises_before_launch(gs, lambda: fwd(d, feat), "packed")
    finally:
        gs[0].tune("gather", 1)

    grads = [torch.empty_like(d[q]) for q in NAMES]
    g_feat = torch.empty_like(feat)
    # a forward without features: no feature backward
    fin, raw, aux, _, _ = rctx.forward_aux(*(d[q] for q in NAMES), *cam)
    gmap = torch.zeros(v.height, v.width, F, device=cuda)
    fake_map = torch.zeros(*raw.shape[:2], F, device=cuda)
    _raises_before_launch(gs, lambda: rctx.backward_feat_into(*(d[q] for q in NAMES), feat, raw, torch.zeros_like(fin),
                                                              True, aux, None, fake_map, gmap, *grads, g_feat),
                          "no features")
    fin, raw, aux, _, fmap, _, _ = fwd(d, feat)

    def bwd(f=feat, gm=gmap):
        rctx.backward_feat_into(*(d[q] for q in NAMES), f, raw, torch.zeros_like(fin), True, aux, None, fmap, gm,
                                *grads, g_feat)

    _raises_before_launch(gs, lambda: bwd(f=feat.clone()), "forward's feature")
    # absgrad statistics with a feature gradient
    st = [torch.zeros(n, device=cuda), torch.zeros(n, dtype=torch.int32, device=cuda), torch.zeros(n, device=cuda),
          torch.zeros(n, device=cuda)]
    rctx.set_densify_stats(st[0], st[1], st[2], st[3])
    _raises_before_launch(gs, bwd, "absgrad")
    rctx.clear_densify_stats()
    # a gradient push: grad_feat is not in the bucket
    bucket = torch.zeros(64, device=cuda)
    staging = [torch.zeros(64, device=cuda) for _ in range(2)]
    rctx.set_grad_push(bucket.data_ptr(), [s.data_ptr() for s in staging], 32, 0)
    _raises_before_launch(gs, bwd, "push")
    rctx.clear_grad_push()
    # the context still works: the same frame differentiates, and NULL grad_map zero-fills grad_feat
    bwd()
    g_feat.fill_(1.0)
    bwd(gm=None)
    torch.cuda.synchronize()
    assert torch.equal(g_feat, torch.zeros_like(g_feat))


def test_feat_loss_reaches_grad2d(gs, cuda):
    """The densification statistic grad2d includes a feature-only loss (its rows are the usual gradient rows)."""
    import renderer
    n, F = 4000, 8
    g, v, _ = scene(n, 128, 96)
    d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
    df = _feat(n, F, 4).to(cuda).requires_grad_(True)
    rctx = gs[0].RenderContext()
    g2, cnt, mr = torch.zeros(n, device=cuda), torch.zeros(n, dtype=torch.int32, device=cuda), torch.zeros(n, device=cuda)
    rctx.set_densify_stats(g2, cnt, mr)
    img, fm, dep, alp, _ = renderer.render_frame_feat(rctx, *(d[q] for q in NAMES), df, *_args(v))
    (fm * torch.linspace(-1, 1, F, device=cuda)).sum().backward()
    torch.cuda.synchronize()
    assert float(g2.max()) > 0 and int(cnt.max()) == 1
    assert float(d["pos"].grad.abs().max()) > 0 and float(df.grad.abs().max()) > 0


@pytest.mark.parametrize("stats", [False, True], ids=["densify", "densify_stats"])
def test_densify_keeps_features_row_aligned(gs, cuda, stats):
    """Every Gaussian gets a unique opacity logit and a feature row encoding it: after prune / clone / split every
    new row's features still match its opacity."""
    n, F = 5000, 16
    g, _, _ = scene(n, 128, 96)
    d = {q: t.to(cuda).contiguous() for q, t in g.items()}
    d["opa"] = torch.linspace(-3, 3, n, device=cuda).reshape(d["opa"].shape).contiguous()
    feat = d["opa"].reshape(n, 1).expand(n, F).contiguous() * torch.arange(1, F + 1, device=cuda)
    gen = torch.Generator().manual_seed(0)
    norm = (d["scale"].abs() + 1e-4).norm(dim=1)
    tau = float(norm.median())
    if stats:
        accum = torch.rand(n, generator=gen).to(cuda)
        count = torch.ones(n, dtype=torch.int32, device=cuda)
        out, counts = gs[0].densify_stats(*(d[q] for q in NAMES), accum, count, None, 0.0, 0, 0.0, 1e9, 0.5, tau,
                                          True, True, feat=feat)
    else:
        grad = (torch.rand(n, 3, generator=gen) * 2 - 1).to(cuda)
        out, counts = gs[0].densify(*(d[q] for q in NAMES), grad, 0, 0.0, 1e9, 0.5, True, tau, True, True, 0.01,
                                    feat=feat)
    assert len(out) == 6 and counts[0] > 0 and counts[1] > 0 and counts[2] > 0, counts
    m = out[0].shape[0]
    assert out[5].shape == (m, F)
    opa = out[2].reshape(m, 1)
    assert torch.equal(out[5], opa * torch.arange(1, F + 1, device=cuda))


def test_feat_full_size_deterministic(gs, cuda):
    """C3 (2.4 M Gaussians, 1080p) at F = 16: forward + backward with image and feature gradients are
    bit-deterministic, the image equals the aux frame's, and the frame launches as many kernels as the aux frame plus
    one (the feature segment sum)."""
    import renderer
    n, w, h, F = 2_400_000, 1920, 1080, 16
    g = {q: t.to(cuda) for q, t in S.make_gaussians(n, w, h, 0).items()}
    v = S.make_view(w, h, 0)
    feat = _feat(n, F, 7).to(cuda)
    gen = torch.Generator().manual_seed(3)
    go = (torch.rand(h, w, 3, generator=gen) * 2 - 1).to(cuda)
    gf = (torch.rand(h, w, F, generator=gen) * 2 - 1).to(cuda)
    rctx = gs[0].RenderContext()
    d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
    img, _, _, _ = renderer.render_frame_aux(rctx, *(d[q] for q in NAMES), *_args(v), background=BG)
    img.backward(go)                               # the first frame of a context also fills its index table
    torch.cuda.synchronize()
    l0 = gs[0].kernel_launches()
    d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
    img, _, _, _ = renderer.render_frame_aux(rctx, *(d[q] for q in NAMES), *_args(v), background=BG)
    img.backward(go)
    torch.cuda.synchronize()
    aux_launches = gs[0].kernel_launches() - l0
    aux_img = img.detach()
    runs, launches = [], []
    for _ in range(2):
        d = {q: t.clone().requires_grad_(True) for q, t in g.items()}
        df = feat.clone().requires_grad_(True)
        l0 = gs[0].kernel_launches()
        img, fm, _, _, _ = renderer.render_frame_feat(rctx, *(d[q] for q in NAMES), df, *_args(v), background=BG)
        torch.autograd.backward([img, fm], [go, gf])
        torch.cuda.synchronize()
        launches.append(gs[0].kernel_launches() - l0)
        runs.append([img.detach(), fm.detach(), df.grad] + [d[q].grad for q in NAMES])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    assert torch.equal(runs[0][0], aux_img)
    assert launches[0] == launches[1] == aux_launches + 1
    assert torch.isfinite(runs[0][2]).all() and float(runs[0][2].abs().max()) > 0


# ------------------------------------------------------------------------------------------
# the Splatter layer: n_features, render_features, densification and checkpoints
def _feature_splatter(g, v, cuda, **kw):
    import splatter
    vs = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)]
    return splatter.Splatter.from_tensors(g, vs, device=cuda, **kw)


def _opa_coded_scene(n, F):
    """Every Gaussian has a unique opacity logit (some below the prune threshold sigmoid^-1(0.02) = -3.9) and a
    feature row that encodes it: feat[i, k] = opa[i] (k + 1)."""
    g, v, _ = scene(n, 128, 96)
    g["opa"] = torch.linspace(-6, 3, n).reshape(g["opa"].shape).contiguous()
    g["feat"] = g["opa"].reshape(n, 1) * torch.arange(1, F + 1, dtype=torch.float32)
    return g, v


def _assert_rows_match_opacity(sp, F):
    gg = sp.gaussian_3ds
    m = gg.pos.shape[0]
    assert tuple(gg.feat.shape) == (m, F) and isinstance(gg.feat, torch.nn.Parameter)
    assert torch.equal(gg.feat.detach(), gg.opa.detach().reshape(m, 1) * torch.arange(1, F + 1, device=gg.feat.device))


def test_splatter_adaptive_control_keeps_features_aligned(gs, cuda):
    n, F = 5000, 16
    g, v = _opa_coded_scene(n, F)
    sp = _feature_splatter(g, v, cuda)
    assert sp.n_features == F
    norm = (sp.gaussian_3ds.scale.detach().abs() + 1e-4).norm(dim=1)
    grad = (torch.rand(n, 3, generator=torch.Generator().manual_seed(0)) * 2 - 1).to(cuda)
    r = sp.gaussian_3ds.adaptive_control(grad, float(norm.median()), 1e9, grad_thresh=0.5)
    assert r["deleted"] > 0 and r["cloned"] > 0 and r["split"] > 0, r
    _assert_rows_match_opacity(sp, F)


def test_splatter_adaptive_control_screen_keeps_features_aligned(gs, cuda):
    n, F = 5000, 8
    g, v = _opa_coded_scene(n, F)
    sp = _feature_splatter(g, v, cuda, n_features=F, densify_stats="grad")
    st = sp.densify_stats
    st.grad2d.copy_(torch.rand(n, generator=torch.Generator().manual_seed(1)).to(cuda))
    st.count.fill_(1)
    norm = (sp.gaussian_3ds.scale.detach().abs() + 1e-4).norm(dim=1)
    r = sp.adaptive_control_screen(float(norm.median()), 1e9, grad_thresh=0.5)
    assert r["deleted"] > 0 and r["cloned"] > 0 and r["split"] > 0, r
    _assert_rows_match_opacity(sp, F)
    out = sp.render_features(0)                                     # the densified scene renders
    assert tuple(out["features"].shape) == (v.height, v.width, F)


def test_splatter_feature_loss_reaches_grad2d(gs, cuda):
    n, F = 4000, 8
    g, v, _ = scene(n, 128, 96)
    sp = _feature_splatter(g, v, cuda, n_features=F, densify_stats="grad")
    gg = sp.gaussian_3ds
    assert torch.equal(gg.feat.detach(), torch.zeros(n, F, device=cuda))   # zero-initialised
    with torch.no_grad():
        gg.feat.copy_(_feat(n, F, 4).to(cuda))
    out = sp.render_features(0, background=BG)
    assert set(out) == {"image", "features", "depth", "alpha"}
    (out["features"] * torch.linspace(-1, 1, F, device=cuda)).sum().backward()
    torch.cuda.synchronize()
    assert float(sp.densify_stats.grad2d.max()) > 0
    assert float(gg.feat.grad.abs().max()) > 0 and float(gg.pos.grad.abs().max()) > 0


def test_checkpoint_round_trip_with_features(gs, cuda, tmp_path):
    import checkpoint
    n, F = 3000, 16
    g, v, _ = scene(n, 96, 64)
    g["feat"] = _feat(n, F, 9)
    sp = _feature_splatter(g, v, cuda)
    path = str(tmp_path / "ckpt.pth")
    sp.save_checkpoint(path)
    saved = torch.load(path, map_location="cpu", weights_only=False)
    assert torch.equal(saved["feat"], g["feat"])
    # Splatter(load_ckpt=...) restores the features (their width comes from the file)
    plain = {k: torch.zeros_like(t) for k, t in g.items() if k != "feat"}
    plain["quat"][:, 0] = 1.0
    sp2 = _feature_splatter(plain, v, cuda, load_ckpt=path)
    assert sp2.n_features == F
    for k in NAMES + ("feat",):
        assert torch.equal(getattr(sp2.gaussian_3ds, k).detach().cpu(), g[k]), k
    # load_checkpoint into a scene with other features replaces them
    other = dict(g, feat=torch.zeros(n, F))
    sp3 = _feature_splatter(other, v, cuda)
    checkpoint.load_checkpoint(path, sp3, restore_rng=False)
    assert torch.equal(sp3.gaussian_3ds.feat.detach().cpu(), g["feat"])
    a = sp2.render_features(0)
    b = sp3.render_features(0)
    assert torch.equal(a["features"], b["features"]) and torch.equal(a["image"], b["image"])


def test_feat_masked_gradient_at_c3(gs, cuda):
    """C3 (2.4 M Gaussians, 1080p) at F = 16: the image and feature upstream gradients are non-zero only on sampled
    tiles (the heaviest, the longest consumed, the most skipped tail, a spread); the feature map on those tiles and
    all six gradients are compared with the fp64 oracle run on exactly the Gaussians the device binned there, and every
    other gradient must be exactly zero."""
    import gs_oracle as O
    from test_scale_parity_gpu import _pick_tiles, _tile_mask
    n, w, h, F = 2_400_000, 1920, 1080, 16
    g, v, cam = scene(n, w, h, k=0)
    g["feat"] = _feat(n, F, 11)
    sp = _feature_splatter(g, v, cuda)
    with torch.no_grad():
        sp.render_features(0)
    st = sp.frame_stats()
    idx, accum = sp._rctx.sorted_instances()
    idx, accum = idx.cpu(), accum.cpu().long()
    neff = sp._rctx.tile_consumed().cpu().long()
    tiles = _pick_tiles(accum, neff, cam.ntx, cam.nty, 5)
    assert st["max_tile_count"] > 1000                 # multi-chunk tiles really are exercised
    mask = _tile_mask(cam, tiles, h, w)
    gen = torch.Generator().manual_seed(12)
    gi = (torch.rand(h, w, 3, generator=gen) * 2 - 1) * mask
    gf = (torch.rand(h, w, F, generator=gen) * 2 - 1) * mask
    out = sp.render_features(0)
    torch.autograd.backward([out["image"], out["features"]], [gi.to(cuda), gf.to(cuda)])

    # fp64 oracle on the Gaussians the device binned into the sampled tiles
    dt = torch.float64
    ids = [idx[int(accum[t]):int(accum[t + 1])].long() for t in tiles]
    U = torch.unique(torch.cat(ids))
    p = {k: g[k][U].to(dt).clone().requires_grad_(True) for k in NAMES + ("feat",)}
    nq, ns, opa_a, rgb_a = O.preactivate(p["quat"], p["scale"], p["opa"], p["rgb"], "abs")
    rp, rc, _ = O.global_culling(p["pos"], nq, ns, cam.rot.to(dt), cam.tran.to(dt), cam.near, cam.half_w, cam.half_h)
    loc = torch.cat([torch.searchsorted(U, i) for i in ids])
    counts = torch.zeros(cam.ntx * cam.nty, dtype=torch.int64)
    for t, i in zip(tiles, ids):
        counts[t] = i.numel()
    acc2 = torch.zeros(counts.numel() + 1, dtype=torch.int64)
    acc2[1:] = torch.cumsum(counts, 0)
    acc2, tt = acc2.to(torch.int32), torch.tensor(tiles)
    opad = O.draw(rp[loc], rgb_a[loc], opa_a[loc], rc[loc], acc2, cam.Hp, cam.Wp, cam.fx, cam.fy, tiles=tt)
    fpad = FT.draw_features(rp[loc], p["feat"][loc], opa_a[loc], rc[loc], acc2, cam.Hp, cam.Wp, cam.fx, cam.fy,
                            tiles=tt)
    torch.autograd.backward([cam.crop(torch.clamp(opad, 0, 1)), cam.crop(fpad)], [gi.to(dt), gf.to(dt)])

    top, left = (cam.Hp - h) // 2, (cam.Wp - w) // 2
    fm = torch.zeros(cam.Hp, cam.Wp, F, dtype=dt)
    fm[top:top + h, left:left + w] = out["features"].detach().cpu().double()
    for t in tiles:
        ty, tx = divmod(t, cam.ntx)
        r0, r1 = max(ty * 16, top), min((ty + 1) * 16, top + h)
        a, b = fm[r0:r1, tx * 16:(tx + 1) * 16], fpad.detach()[r0:r1, tx * 16:(tx + 1) * 16]
        assert abs_err(a, b) < 1e-4 * max(1.0, float(g["feat"].abs().max())), t
    other = torch.ones(n, dtype=torch.bool)
    other[U] = False
    for name in NAMES + ("feat",):
        got = getattr(sp.gaussian_3ds, name).grad.cpu()
        assert bool(torch.isfinite(got).all()), name
        assert rel_err(got[U], p[name].grad) < GRAD_RTOL, (name, rel_err(got[U], p[name].grad))
        assert float(got[other].abs().max()) == 0.0, name


def test_feat_misaligned_upstream_gradient(gs, cuda):
    """A contiguous but not 16-byte aligned feature gradient (a narrow view of a larger buffer) is accepted."""
    import renderer
    n, F = 2000, 8
    g, v, _ = scene(n, 96, 64)
    d = {q: t.to(cuda).clone().requires_grad_(True) for q, t in g.items()}
    df = _feat(n, F, 2).to(cuda).requires_grad_(True)
    rctx = gs[0].RenderContext()
    img, fm, _, _, _ = renderer.render_frame_feat(rctx, *(d[q] for q in NAMES), df, *_args(v))
    up = torch.rand(fm.numel() + 1, device=cuda)[1:].view(fm.shape)
    assert up.is_contiguous() and up.data_ptr() % 16
    fm.backward(up)
    ref = df.grad.clone()
    df.grad = None
    img, fm, _, _, _ = renderer.render_frame_feat(rctx, *(d[q] for q in NAMES), df, *_args(v))
    fm.backward(up.clone())
    assert torch.equal(df.grad, ref)
