"""A batch of camera views rendered as one fused frame (renderer.render_frame_batch, gs_render_forward_batch /
gs_render_backward_batch): every view's slice equals a single-view render_frame_aux of that view bit for bit, the
parameter gradients equal the single-view gradients (bit for bit for one view, summed in view order to 1e-6 relative
for several), against the fp64 oracle, the densification statistics, the 4-byte tile-key path, the launch count and
the refusals."""
import math

import pytest
import torch

import filter_oracle as F
import gs_oracle as O
import sh_gaussian_oracle as G
import synthetic as S
from helpers import abs_err, device_depth_keys, rel_err, scene

pytestmark = pytest.mark.gpu

NAMES = ("pos", "rgb", "opa", "quat", "scale")
BG = (0.2, 0.5, 0.9)


def _view(w, h, k=0, focal=1.0, tran=None, rot=None):
    v = S.make_view(w, h, k)
    return dict(fx=v.fx * focal, fy=v.fy * focal * (1.1 if focal != 1.0 else 1.0),
                rot=v.rot if rot is None else rot, tran=v.tran if tran is None else torch.tensor(tran),
                near=v.near)


def _hetero_views(w, h):
    """four poses and focal lengths: a plain one, a zoomed orbit view, one looking away from the scene (no instances),
    one shifted so that part of the scene is culled"""
    return [_view(w, h, 0), _view(w, h, 1, focal=1.3), _view(w, h, 0, tran=(0.0, 0.0, -4.0)),
            _view(w, h, 2, focal=0.8, tran=(1.6, 0.4, 4.0))]


def _params(g, dev):
    return {q: t.to(dev).clone().requires_grad_(True) for q, t in g.items()}


def _upstream(b, rows, cols, seed):
    gen = torch.Generator().manual_seed(seed)
    return ((torch.rand(b, rows, cols, 3, generator=gen) * 2 - 1), (torch.rand(b, rows, cols, generator=gen) * 2 - 1),
            (torch.rand(b, rows, cols, generator=gen) * 2 - 1))


def _single(gs, rctx, g, w, h, views, final, bg, up, dev, use_maps=True):
    """per-view render_frame_aux outputs, M and gradients; the gradients summed in view order as autograd accumulates"""
    _, renderer = gs
    outs, ms, total = [], [], None
    for v, vw in enumerate(views):
        p = _params(g, dev)
        img, dep, alp, mask = renderer.render_frame_aux(rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], w,
                                                        h, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"],
                                                        0.05, "abs", background=bg, final=final)
        ms.append(rctx.last_instances())
        outs.append((img.detach(), dep.detach(), alp.detach(), mask))
        ys = [img, dep, alp] if use_maps else [img]
        gr = torch.autograd.grad(ys, [p[q] for q in NAMES], [u[v].to(dev) for u in up][:len(ys)])
        total = list(gr) if total is None else [a + b for a, b in zip(total, gr)]
    return outs, ms, total


def _batch(gs, rctx, g, w, h, views, final, bg, up, dev, use_maps=True):
    _, renderer = gs
    p = _params(g, dev)
    img, dep, alp, mask = renderer.render_frame_batch(
        rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], w, h, [vw["fx"] for vw in views],
        [vw["fy"] for vw in views], torch.stack([vw["rot"] for vw in views]), torch.stack([vw["tran"] for vw in views]),
        views[0]["near"], 0.05, "abs", background=bg, final=final)
    m = rctx.last_instances()
    ys = [img, dep, alp] if use_maps else [img]
    gr = torch.autograd.grad(ys, [p[q] for q in NAMES], [u.to(dev) for u in up][:len(ys)])
    return (img.detach(), dep.detach(), alp.detach(), mask), m, list(gr)


def _setup(gs, sh_dim, filt):
    gaussian, renderer = gs
    rctx = gaussian.RenderContext()
    if sh_dim != 3:
        rctx.set_sh_eval(renderer.SH_EVAL["gaussian"])
    rctx.set_filter2d(renderer.FILTER2D[filt], 0.3)
    return rctx


def _shape(w, h, final):
    return (h, w) if final else (int(math.ceil(h / 16)) * 16, int(math.ceil(w / 16)) * 16)


@pytest.mark.parametrize("final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("sh_dim,filt", [(3, "none"), (3, "dilate"), (3, "antialias"), (27, "none"), (48, "antialias")])
def test_one_view_equals_single_frame_bitwise(gs, cuda, sh_dim, filt, final):
    w, h = 200, 120
    g, _, _ = scene(6000, w, h, k=0, sh_dim=sh_dim)
    views = [_view(w, h, 1, focal=1.2)]
    up = _upstream(1, *_shape(w, h, final), 3)
    rctx = _setup(gs, sh_dim, filt)
    so, sm, sg = _single(gs, rctx, g, w, h, views, final, BG, up, cuda)
    bo, bm, bg_ = _batch(gs, rctx, g, w, h, views, final, BG, up, cuda)
    assert bm == sm[0] > 0
    for a, b in zip(bo, so[0]):
        assert torch.equal(a[0], b)
    for q, a, b in zip(NAMES, bg_, sg):
        assert torch.equal(a, b), q


@pytest.mark.parametrize("grad_is_final", [True, False], ids=["final", "padded"])
@pytest.mark.parametrize("sh_dim,filt,use_maps", [(3, "none", True), (3, "antialias", False), (48, "dilate", True)])
def test_heterogeneous_views_equal_single_frames(gs, cuda, sh_dim, filt, use_maps, grad_is_final):
    w, h = 184, 120
    g, _, _ = scene(8000, w, h, k=0, sh_dim=sh_dim)
    views = _hetero_views(w, h)
    up = _upstream(4, *_shape(w, h, grad_is_final), 7)
    rctx = _setup(gs, sh_dim, filt)
    so, sm, sg = _single(gs, rctx, g, w, h, views, grad_is_final, BG, up, cuda, use_maps)
    bo, bm, bg_ = _batch(gs, rctx, g, w, h, views, grad_is_final, BG, up, cuda, use_maps)
    assert sm[2] == 0 and min(sm[0], sm[1], sm[3]) > 0          # the view looking away has no instance
    assert so[3][3].sum() < so[0][3].sum()                       # the shifted view culls part of the scene
    assert bm == sum(sm)
    for v in range(4):
        for a, b in zip(bo, so[v]):
            assert torch.equal(a[v], b), v
    for q, a, b in zip(NAMES, bg_, sg):
        assert rel_err(a, b) <= 1e-6, q


@pytest.mark.parametrize("sh_dim,filt", [(3, "none"), (3, "antialias"), (27, "dilate")])
def test_batch_vs_oracle(gs, cuda, sh_dim, filt):
    w, h = 128, 96
    g, _, _ = scene(3000, w, h, k=0, sh_dim=sh_dim)
    views = [_view(w, h, 0), _view(w, h, 1, focal=1.25), _view(w, h, 7, focal=0.9)]
    up = _upstream(3, h, w, 11)
    rctx = _setup(gs, sh_dim, filt)
    bo, _, bgr = _batch(gs, rctx, g, w, h, views, True, BG, up, cuda)
    p = {q: t.double().clone().requires_grad_(True) for q, t in g.items()}
    ref_img, ref_grad = [], None
    for v, vw in enumerate(views):
        cam = O.Camera(w, h, vw["fx"], vw["fy"], vw["rot"], vw["tran"], vw["near"])
        rgb = G.gaussian_logits(p["pos"], p["rgb"], cam) if sh_dim != 3 else p["rgb"]
        o = F.render_maps(p["pos"], rgb, p["opa"], p["quat"], p["scale"], cam, mode=filt, variance=0.3, background=BG,
                          depth_key=device_depth_keys(g, cam, cuda))
        ref_img.append(o["image"])
        gr = torch.autograd.grad([o["image"], o["depth"], o["alpha"]], [p[q] for q in NAMES],
                                 [up[0][v].double(), up[1][v].double(), up[2][v].double()], allow_unused=True)
        gr = [torch.zeros_like(p[q]) if t is None else t for q, t in zip(NAMES, gr)]
        ref_grad = gr if ref_grad is None else [a + b for a, b in zip(ref_grad, gr)]
    for v in range(3):
        assert abs_err(bo[0][v], ref_img[v]) < 1e-4, v
    for q, a, b in zip(NAMES, bgr, ref_grad):
        assert rel_err(a, b) < 1e-3, q


@pytest.mark.parametrize("absgrad", [False, True], ids=["grad", "absgrad"])
def test_densify_stats_equal_single_backwards(gs, cuda, absgrad):
    w, h = 184, 120
    n = 8000
    g, _, _ = scene(n, w, h, k=0)
    views = _hetero_views(w, h)
    up = _upstream(4, h, w, 5)

    def stats():
        return [torch.zeros(n, device=cuda), torch.zeros(n, dtype=torch.int32, device=cuda),
                torch.zeros(n, device=cuda), torch.zeros(n, device=cuda) if absgrad else None]

    res = []
    for runner in (_single, _batch):
        rctx = _setup(gs, 3, "none")
        st = stats()
        rctx.set_densify_stats(*st)
        runner(gs, rctx, g, w, h, views, True, None, up, cuda)
        torch.cuda.synchronize()
        res.append(st)
    (g2s, cs, rs, as_), (g2b, cb, rb, ab) = res
    assert torch.equal(cs, cb) and torch.equal(rs, rb) and int(cb.max()) >= 2
    assert rel_err(g2b, g2s) <= 1e-6
    if absgrad:
        assert rel_err(ab, as_) <= 1e-6


def test_four_byte_tile_keys(gs, cuda):
    """9 views at 1920x1080: B T = 73,440 tiles > 65,536, so the tile sort runs on 4-byte keys"""
    w, h = 1920, 1080
    g, _, _ = scene(20000, w, h, k=0)
    views = [_view(w, h, k % 8, focal=1.0 + 0.05 * k) for k in range(9)]
    up = _upstream(9, h, w, 2)
    rctx = _setup(gs, 3, "none")
    bo, bm, bgr = _batch(gs, rctx, g, w, h, views, True, None, up, cuda, use_maps=False)
    so, sm, sg = _single(gs, rctx, g, w, h, views, True, None, up, cuda, use_maps=False)
    assert bm == sum(sm)
    for v in range(9):
        for a, b in zip(bo, so[v]):
            assert torch.equal(a[v], b), v
    for q, a, b in zip(NAMES, bgr, sg):
        assert rel_err(a, b) <= 1e-6, q


def test_launch_count_independent_of_batch(gs, cuda):
    gaussian, renderer = gs
    w, h = 160, 96
    g, _, _ = scene(4000, w, h, k=0)
    rctx = _setup(gs, 3, "none")
    counts = {}
    for b in (1, 4, 8, 0):
        views = [_view(w, h, k % 8) for k in range(max(b, 1))]
        up = _upstream(len(views), h, w, 1)
        run = (lambda: _single(gs, rctx, g, w, h, views, True, BG, up, cuda)) if b == 0 else \
            (lambda: _batch(gs, rctx, g, w, h, views, True, BG, up, cuda))
        run()                                                     # warm-up: workspaces, the iota of the depth sort
        torch.cuda.synchronize()
        k0 = gaussian.kernel_launches()
        run()
        torch.cuda.synchronize()
        counts[b] = gaussian.kernel_launches() - k0
    assert counts[1] == counts[4] == counts[8] == counts[0], counts


def _expect_refused(gaussian, fn, text):
    k0 = gaussian.kernel_launches()
    with pytest.raises(RuntimeError, match=text):
        fn()
    assert gaussian.kernel_launches() == k0


def test_refusals_before_any_launch(gs, cuda):
    gaussian, renderer = gs
    w, h = 96, 64
    g, _, _ = scene(1000, w, h, k=0)
    gsh, _, _ = scene(1000, w, h, k=0, sh_dim=27)
    p = {q: t.to(cuda) for q, t in g.items()}
    psh = {q: t.to(cuda) for q, t in gsh.items()}
    views = [_view(w, h, 0), _view(w, h, 1)]
    focal = torch.tensor([[vw["fx"], vw["fy"]] for vw in views], dtype=torch.float64)
    rot = torch.stack([vw["rot"] for vw in views])
    tran = torch.stack([vw["tran"] for vw in views])
    rctx = gaussian.RenderContext()

    def fwd(params=p, f=focal, r=rot, t=tran, wd=w):
        return rctx.forward_batch(params["pos"], params["rgb"], params["opa"], params["quat"], params["scale"], wd, h,
                                  f, r, t, 0.3, 0.05, 0, None, True)

    # per-pixel SH colour
    _expect_refused(gaussian, lambda: fwd(psh), r"\(-2\).*per pixel")
    # the packed path, and a non-default blend knob
    for knob, val in (("gather", 0), ("blend_repack", 0), ("bwd_unroll", 2)):
        gaussian.tune(knob, val)
        try:
            _expect_refused(gaussian, fwd, r"\(-2\)")
        finally:
            gaussian.tune(knob, {"gather": 1, "blend_repack": 1, "bwd_unroll": 4}[knob])
    # n_views out of range (the binding checks the shapes before the C entry point)
    big = 65
    _expect_refused(gaussian, lambda: fwd(f=focal[:1].repeat(big, 1), r=rot[:1].repeat(big, 1, 1),
                                          t=tran[:1].repeat(big, 1)), "1 <= B")
    with pytest.raises(ValueError):
        renderer.render_frame_batch(rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], w, h, [1.0] * big,
                                    [1.0] * big, rot[:1].repeat(big, 1, 1), tran[:1].repeat(big, 1), 0.3, 0.05, "abs")
    with pytest.raises(ValueError):
        renderer.render_frame_batch(rctx, p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], w, h, [1.0],
                                    [1.0, 2.0], rot[:1], tran[:1], 0.3, 0.05, "abs")
    # a batch whose tile rows overflow the rectangle's 16-bit row field: B Hp / 16 = 64 * 1024 > 65535
    tall = 16 * 1024
    _expect_refused(gaussian, lambda: rctx.forward_batch(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], 16, tall,
                                                         focal[:1].repeat(64, 1), rot[:1].repeat(64, 1, 1),
                                                         tran[:1].repeat(64, 1), 0.3, 0.05, 0, None, False),
                    r"\(-1\).*65535")
    # a data-parallel gradient push configured
    bucket = torch.zeros(1024, device=cuda)
    staging = [torch.zeros(1024, device=cuda) for _ in range(2)]

    def push():
        rctx.set_grad_push(bucket.data_ptr(), [t.data_ptr() for t in staging], 512, 0)

    push()
    try:
        _expect_refused(gaussian, fwd, r"\(-2\).*push")
    finally:
        rctx.clear_grad_push()
    # every single-view backward entry after a batched forward
    fin, raw, aux, aux_fin, _ = fwd()
    torch.cuda.synchronize()
    outs = [torch.empty_like(p[q]) for q in NAMES]
    args = (p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"])
    feat = torch.zeros(p["pos"].shape[0], 8, device=cuda)
    fmap = torch.zeros(*raw.shape[1:3], 8, device=cuda)
    single = {
        "plain": lambda: rctx.backward_into(*args, raw[0], torch.zeros_like(raw[0]), *outs, -1),
        "final": lambda: rctx.backward_final_into(*args, raw[0], torch.zeros_like(fin[0]), *outs, -1),
        "aux": lambda: rctx.backward_aux_into(*args, raw[0], torch.zeros_like(fin[0]), True, aux[0], None, *outs, -1),
        "cam": lambda: rctx.backward_cam_into(*args, raw[0], torch.zeros_like(fin[0]), True, aux[0], None, *outs,
                                              torch.zeros(12, device=cuda), -1),
        "feat": lambda: rctx.backward_feat_into(*args, feat, raw[0], torch.zeros_like(fin[0]), True, aux[0], None, fmap,
                                                None, *outs, torch.empty_like(feat), -1),
    }
    for name, fn in single.items():
        _expect_refused(gaussian, fn, r"\(-1\).*batched")
    # a gradient push configured between a batched forward and its backward
    push()
    try:
        _expect_refused(gaussian, lambda: rctx.backward_batch_into(*args, raw, torch.zeros_like(fin), True, aux, None,
                                                                   *outs, -1), r"\(-2\).*push")
    finally:
        rctx.clear_grad_push()
    # the batched backward after a single-view forward
    rctx.forward_aux(*args, w, h, views[0]["fx"], views[0]["fy"], rot[0], tran[0], 0.3, 0.05, 0, None, True)
    torch.cuda.synchronize()
    _expect_refused(gaussian, lambda: rctx.backward_batch_into(*args, raw, torch.zeros_like(fin), True, aux, None,
                                                               *outs, -1), r"\(-1\).*not batched")


def _splatter_scene(cuda, n, w, h, k, **kw):
    import splatter
    g = S.make_gaussians(n, w, h, 5, 3, (0.05, 0.9), (0.6, 5.0))
    views = [S.make_view(w, h, j) for j in range(k)]
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    return g, views, splatter.Splatter.from_tensors(g, vd, device=cuda, **kw)


def test_splatter_batch_training_lowers_the_loss(gs, cuda):
    """a few mini-batch steps of 4 views against targets rendered from a perturbed scene"""
    w, h = 128, 96
    g, views, target_sp = _splatter_scene(cuda, 3000, w, h, 4)
    with torch.no_grad():
        targets = target_sp.render_batch(range(4))["image"].detach()
        for q in ("pos", "rgb"):
            getattr(target_sp.gaussian_3ds, q).add_(0.05 * torch.randn_like(getattr(target_sp.gaussian_3ds, q)))
    sp = target_sp
    opt = torch.optim.Adam(sp.gaussian_3ds.parameters(), lr=1e-2)
    losses = []
    for _ in range(8):
        out = sp.render_batch(range(4))
        loss = (out["image"] - targets).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert out["image"].shape == (4, h, w, 3) and out["culling_mask"].shape == (4, 3000)
    assert torch.equal(sp.culling_mask, out["culling_mask"].sum(0))
    assert losses[-1] < 0.8 * losses[0], losses


def test_splatter_adaptive_control_after_batched_backwards(gs, cuda):
    w, h = 128, 96
    _, _, sp = _splatter_scene(cuda, 3000, w, h, 4, densify_stats="grad")
    for _ in range(2):
        out = sp.render_batch([0, 1, 2, 3])
        out["image"].sum().backward()
    st = sp.densify_stats
    assert int(st.count.max()) == 8
    thr = float((st.grad2d / st.count.clamp(min=1)).quantile(0.8))
    tau = float(sp.gaussian_3ds.scale.detach().norm(dim=-1).median())
    info = sp.adaptive_control_screen(tau, 10.0, grad_thresh=thr)
    assert info["cloned"] + info["split"] > 0 and sp.gaussian_3ds.pos.shape[0] == info["total"]
    out = sp.render_batch([0, 1, 2, 3])
    out["image"].sum().backward()
    assert torch.isfinite(sp.gaussian_3ds.pos.grad).all()


def test_splatter_batch_c3_full_size(gs, cuda):
    """the C3 scene at 1920x1080, four views: finite, each slice equal to a single-view render, M the sum"""
    w, h = 1920, 1080
    _, _, sp = _splatter_scene(cuda, 2_400_000, w, h, 4)
    with torch.no_grad():
        out = sp.render_batch(range(4))
        m = sp.n_tile_gaussians
        assert torch.isfinite(out["image"]).all()
        ms = []
        for v in range(4):
            single = sp.render_maps(v)
            ms.append(sp.n_tile_gaussians)
            assert torch.equal(out["image"][v], single["image"]), v
            assert torch.equal(out["depth"][v], single["depth"]), v
    assert m == sum(ms)
    with pytest.raises(ValueError):
        import splatter
        bad = splatter.Splatter.from_tensors(
            S.make_gaussians(100, 64, 48, 0), [dict(width=64, height=48, focal_x=50.0, focal_y=50.0,
                                                    rot=torch.eye(3), tran=torch.tensor([0.0, 0.0, 4.0])),
                                               dict(width=32, height=48, focal_x=50.0, focal_y=50.0,
                                                    rot=torch.eye(3), tran=torch.tensor([0.0, 0.0, 4.0]))],
            device=cuda)
        bad.render_batch([0, 1])
