"""Blend-weight scores (gs_frame_scores, RenderContext.scores_into, Splatter.score_views / accumulate_scores) and
Splatter.prune on the device: against the fp64 oracle of tests/scores_oracle.py for every frame kind, on the edge
scenes of tests/tile_edges.py, the invariants (alpha map sum, determinism, batched = single views, no effect on the
backward), the refusals that need a context, and pruning (bit-identical frames, feature rows, optimizer moments, the
trainer)."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

import scores_oracle as SO
import tile_edges as E
from helpers import device_depth_keys, scene

pytestmark = pytest.mark.gpu

TOL = 1e-4
NAMES = ("pos", "rgb", "opa", "quat", "scale")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENSES = {"opencv": dict(model="OPENCV", k=[-0.08, 0.01, 0.002, -0.001]),
          "fisheye": dict(model="FISHEYE", k=[0.05, -0.01, 0.0, 0.0])}


def _views(vs, lens=None):
    out = []
    for v in vs:
        d = dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran)
        if lens is not None:
            d["lens"] = dict(lens, cx=v.width / 2 + 3.5, cy=v.height / 2 - 2.0)
        out.append(d)
    return out


def _splatter(g, vs, dev, lens=None, **kw):
    import splatter
    return splatter.Splatter.from_tensors(g, _views(vs, lens), device=dev, near=vs[0].near,
                                          use_sh_coeff=g["rgb"].shape[1] != 3, **kw)


def _scores(sp):
    import splatter
    return splatter.ContributionScores(sp.gaussian_3ds.pos.shape[0], sp.device)


def _check(got, ref, label=""):
    ws, wm, npix = ref
    gs_, gm = got.weight_sum.double().cpu(), got.weight_max.double().cpu()
    bad_s = (gs_ - ws).abs() > TOL * npix.clamp(min=1)
    bad_m = (gm - wm).abs() > TOL
    assert not bool(bad_s.any()), (label, int(bad_s.sum()), float((gs_ - ws).abs().max()))
    assert not bool(bad_m.any()), (label, int(bad_m.sum()), float((gm - wm).abs().max()))
    assert float(ws.sum()) > 0


KINDS = ["rgb", "sh27-gauss", "sh48-gauss", "sh27-pixel-tc0", "sh48-pixel-tc3", "dilate", "antialias", "filter3d",
         "opencv", "fisheye", "feat16"]


@pytest.mark.parametrize("kind", KINDS)
def test_scores_vs_oracle(gs, cuda, kind):
    sh = int(kind[2:4]) if kind.startswith("sh") else 3
    g, v, cam = scene(3000, 120, 88, k=1, sh_dim=sh)
    kw = {}
    if kind.startswith("sh"):
        kw["sh_eval"] = "gaussian" if kind.endswith("gauss") else "pixel"
    if kind in ("dilate", "antialias"):
        kw["filter2d"] = kind
    if kind == "filter3d":
        kw["filter3d"] = True
    if kind.startswith("feat"):
        kw["n_features"] = 16
    tc = int(kind[-1]) if "-tc" in kind else None
    lens = LENSES.get(kind)
    keys = device_depth_keys(g, cam, cuda)
    if lens is not None:                     # away from ties of fp32 and fp64 at rho_max, the frustum and tile edges
        import test_lens_gpu as TL
        g = TL._stable(g, cam, dict(lens, cx=v.width / 2 + 3.5, cy=v.height / 2 - 2.0))
        keys = TL._depth_keys(g, cam, cuda)
    sp = _splatter(g, [v], cuda, lens=lens, **kw)
    try:
        if tc is not None:
            gs[0].tune("sh_tc", tc)
        with torch.no_grad():
            sp.render_features(0) if kind.startswith("feat") else sp(0)
        got = sp.accumulate_scores(_scores(sp))
    finally:
        if tc is not None:
            gs[0].tune("sh_tc", -1)
    gref = dict(g)
    if kind == "filter3d":                                     # the filter folded into opacity and scale in fp64
        opa, scale = sp.bake_filter3d()
        gref = dict(g, opa=opa.cpu(), scale=scale.cpu())
    ln = None if lens is None else sp.views[0]["lens"]
    ref = SO.scores(gref, cam, mode=kw.get("filter2d", "none"), lens=ln, depth_key=keys)
    _check(got, ref, kind)


def test_batch_scores_vs_oracle_and_single_views(gs, cuda):
    """score_views over 3 views (one batched frame) against the oracle summed over the views, and bit for bit against
    three single-view frames each scored in view order."""
    g, _, _ = scene(3000, 120, 88, k=0)
    vs = [scene(1, 120, 88, k=k)[1] for k in range(3)]
    sp = _splatter(g, vs, cuda)
    got = sp.score_views(batch_size=8)
    ws = wm = npix = 0
    for v in vs:
        cam = E.O.Camera(v.width, v.height, v.fx, v.fy, v.rot, v.tran, v.near)
        s, m, p = SO.scores(g, cam, depth_key=device_depth_keys(g, cam, cuda))
        ws, npix = ws + s, npix + p
        wm = m if isinstance(wm, int) else torch.maximum(wm, m)
    _check(got, (ws, wm, npix), "batch")
    one = _scores(sp)
    with torch.no_grad():
        for k in range(3):
            sp(k)
            sp.accumulate_scores(one)
    assert torch.equal(one.weight_sum, got.weight_sum) and torch.equal(one.weight_max, got.weight_max)


@pytest.mark.parametrize("name", list(E.BUILDERS))
def test_edge_scenes_vs_oracle(gs, cuda, name):
    """Chunk boundaries, early stops on a chunk edge, walls and depth ties (tests/tile_edges.py)."""
    fx = E.BUILDERS[name]()
    sp = _splatter(fx.g, [fx.view], cuda)
    with torch.no_grad():
        sp(0)
    got = sp.accumulate_scores(_scores(sp))
    _check(got, SO.scores(fx.g, fx.cam, depth_key=device_depth_keys(fx.g, fx.cam, cuda)), name)


def test_no_stale_rows_after_a_frame_with_more_instances(gs, cuda):
    """The walls scene scored right after the same geometry with weaker walls (its tiles stop later, so more rows are
    tagged): the earlier pass's rows must not reach the scores."""
    fx = E.BUILDERS["walls"]()
    weak = torch.where(fx.tile_of < 0, torch.full_like(fx.g["opa"], -0.5), fx.g["opa"])
    sp = _splatter(dict(fx.g, opa=weak), [fx.view], cuda)
    with torch.no_grad():
        sp(0)
        sp.accumulate_scores(_scores(sp))
        sp.gaussian_3ds.opa.copy_(fx.g["opa"].to(cuda))
        sp(0)
    got = sp.accumulate_scores(_scores(sp))
    _check(got, SO.scores(fx.g, fx.cam, depth_key=device_depth_keys(fx.g, fx.cam, cuda)), "stale")


def test_weight_sum_equals_the_alpha_map_and_runs_are_equal(gs, cuda):
    g, v, cam = scene(20000, 320, 200, k=2)
    sp = _splatter(g, [v], cuda)
    with torch.no_grad():
        alpha = sp.render_maps(0)["alpha"]
    a = sp.accumulate_scores(_scores(sp))
    b = sp.accumulate_scores(_scores(sp))
    assert torch.equal(a.weight_sum, b.weight_sum) and torch.equal(a.weight_max, b.weight_max)
    twice = sp.accumulate_scores(sp.accumulate_scores(_scores(sp)))
    assert torch.equal(twice.weight_sum, a.weight_sum + a.weight_sum)
    sa, sw = float(alpha.double().sum()), float(a.weight_sum.double().sum())
    assert abs(sa - sw) <= 1e-5 * sa, (sa, sw)


def test_scores_leave_the_backward_alone(gs, cuda):
    """forward, scores, backward gives the gradients and densification statistics of forward, backward, bit for bit."""
    g, v, cam = scene(8000, 200, 136, k=1)
    out = []
    for score in (False, True):
        sp = _splatter(g, [v], cuda, densify_stats="absgrad")
        img = sp(0)
        if score:
            sp.accumulate_scores(_scores(sp))
        (img * torch.linspace(0, 1, img.numel(), device=cuda).reshape(img.shape)).sum().backward()
        gg = sp.gaussian_3ds
        st = sp.densify_stats
        out.append([getattr(gg, q).grad.clone() for q in NAMES] + [st.grad2d.clone(), st.absgrad.clone(),
                                                                  st.count.clone(), st.max_radius.clone()])
    for x, y in zip(*out):
        assert torch.equal(x, y)


def _refused(gs, fn, exc=RuntimeError, match=None):
    """fn raises before any launch of the library's kernels."""
    n0 = gs[0].kernel_launches()
    with pytest.raises(exc, match=match):
        fn()
    assert gs[0].kernel_launches() == n0


def test_refusals_with_a_context(gs, cuda):
    rctx = gs[0].RenderContext()
    ws, wm = torch.zeros(10, device=cuda), torch.zeros(10, device=cuda)
    _refused(gs, lambda: rctx.scores_into(ws, wm), match="no forward")
    g, v, cam = scene(500, 64, 48)
    sp = _splatter(g, [v], cuda)
    with torch.no_grad():
        sp(0)
    _refused(gs, lambda: sp._rctx.scores_into(ws, wm), match="n differs")
    _refused(gs, lambda: sp._rctx.scores_into(torch.zeros(500, device=cuda, dtype=torch.float64),
                                              torch.zeros(500, device=cuda)), match="float32")
    su = _splatter(g, [v], cuda, primitive="surfel")
    with torch.no_grad():
        su(0)
    _refused(gs, lambda: su._rctx.scores_into(torch.zeros(500, device=cuda), torch.zeros(500, device=cuda)),
             match="surfels")
    _refused(gs, lambda: su.score_views(), ValueError)
    _refused(gs, lambda: su.accumulate_scores(_scores(su)), ValueError)
    try:
        gs[0].tune("gather", 0)
        with torch.no_grad():
            sp(0)
        _refused(gs, lambda: sp.accumulate_scores(_scores(sp)), match="packed path")
    finally:
        gs[0].tune("gather", 1)


class _Scores(ctypes.Structure):
    _fields_ = [("n", ctypes.c_int), ("weight_sum", ctypes.c_void_p), ("weight_max", ctypes.c_void_p)]


def test_c_refusals_with_a_context(gs, cuda):
    """gs_frame_scores on a live context: a null struct, a null weight_sum or weight_max (whatever the forward state),
    and no forward yet are GS_ERR_INVALID_ARG with gs_last_error set and no launch."""
    lib = ctypes.CDLL(os.path.join(ROOT, "3d-gaussian-splatting_b200", "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    lib.gs_kernel_launches.restype = ctypes.c_ulonglong
    lib.gs_ctx_create.argtypes = [ctypes.POINTER(ctypes.c_void_p)]
    lib.gs_ctx_destroy.argtypes = [ctypes.c_void_p]
    lib.gs_frame_scores.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    torch.cuda.set_device(cuda)
    ctx = ctypes.c_void_p()
    assert lib.gs_ctx_create(ctypes.byref(ctx)) == 0
    buf = torch.zeros(2, 16, device=cuda)
    a, b = buf[0].data_ptr(), buf[1].data_ptr()
    try:
        for s, what in ((None, "null argument"), (_Scores(16, None, b), "null argument"),
                        (_Scores(16, a, None), "null argument"), (_Scores(0, None, None), "null argument"),
                        (_Scores(16, a, b), "no forward")):
            before = lib.gs_kernel_launches()
            assert lib.gs_frame_scores(ctx, None if s is None else ctypes.byref(s), None) == -1
            msg = lib.gs_last_error().decode()
            assert "gs_frame_scores" in msg and what in msg, msg
            assert lib.gs_kernel_launches() == before
    finally:
        lib.gs_ctx_destroy(ctx)


def test_score_views_after_a_gradient_push_keeps_the_frame_attributes(gs, cuda):
    """A context left with a data-parallel push by earlier backwards (batched frames refuse one): score_views clears it
    and scores as a fresh context does; the Splatter's last-frame attributes are those of the frame before it."""
    g, _, _ = scene(3000, 120, 88, k=0)
    vs = [scene(1, 120, 88, k=k)[1] for k in range(3)]
    ref = _splatter(g, vs, cuda).score_views()
    sp = _splatter(g, vs, cuda)
    with torch.no_grad():
        sp(1)
    before = (sp.culling_mask.clone(), sp.n_tile_gaussians, sp.current_view, sp.tile_info)
    arena = torch.zeros(3 * 64, device=cuda)
    sp._rctx.set_grad_push(arena.data_ptr(), [arena[64:].data_ptr(), arena[128:].data_ptr()], 32, 0)
    with pytest.raises(RuntimeError, match="gradient push"):
        sp.render_batch([0, 1])
    sp._rctx.set_grad_push(arena.data_ptr(), [arena[64:].data_ptr(), arena[128:].data_ptr()], 32, 0)
    got = sp.score_views()
    assert torch.equal(got.weight_sum, ref.weight_sum) and torch.equal(got.weight_max, ref.weight_max)
    assert torch.equal(sp.culling_mask, before[0]) and sp.n_tile_gaussians == before[1]
    assert sp.current_view is before[2] and sp.tile_info is before[3]


def _kept(g, keep):
    k = keep.cpu()
    return {q: t[k].contiguous() for q, t in g.items()}


def test_prune_matches_a_scene_built_from_the_kept_rows(gs, cuda):
    import splatter
    g, v, cam = scene(6000, 160, 120, k=1)
    feat = torch.rand(6000, 8)
    sp = _splatter(dict(g, feat=feat), [v], cuda)
    sc = sp.score_views()
    k = 3000
    keep = torch.zeros(6000, dtype=torch.bool, device=cuda).index_fill_(
        0, torch.sort(sc.weight_sum, descending=True, stable=True).indices[:k], True)
    assert sp.prune(keep) == 3000 and sp.gaussian_3ds.pos.shape[0] == 3000
    ref = _splatter(_kept(dict(g, feat=feat), keep), [v], cuda)
    assert torch.equal(sp.gaussian_3ds.feat.detach().cpu(), feat[keep.cpu()])
    out = []
    for s in (sp, ref):
        img = s(0)
        (img * torch.linspace(-1, 1, img.numel(), device=cuda).reshape(img.shape)).sum().backward()
        out.append([img.detach()] + [getattr(s.gaussian_3ds, q).grad for q in NAMES])
    for x, y in zip(*out):
        assert torch.equal(x, y)
    with pytest.raises(ValueError):
        sp.prune(torch.zeros(3000, dtype=torch.bool, device=cuda))


def _train_steps(sp, opt, steps=2, visible=False):
    for k in range(steps):
        opt.zero_grad(set_to_none=True)
        img = sp(k % len(sp.views))
        (img - 0.5).abs().mean().backward()
        opt.step(visible=sp.visible_mask()) if visible else opt.step()


def _opt(sp, cls):
    g = sp.gaussian_3ds
    return cls([{"params": g.opa, "lr": 0.03}, {"params": g.rgb, "lr": 0.03}, {"params": g.pos, "lr": 0.003},
                {"params": g.scale, "lr": 0.003}, {"params": g.quat, "lr": 0.003}], betas=(0.9, 0.99))


@pytest.mark.parametrize("mode", ["flat-dense", "flat-visible", "torch"])
def test_prune_keeps_the_kept_moments(gs, cuda, mode):
    import optim
    g, v, cam = scene(4000, 128, 96, k=1)
    v2 = scene(1, 128, 96, k=3)[1]
    sp = _splatter(g, [v, v2], cuda)
    opt = _opt(sp, torch.optim.Adam if mode == "torch" else optim.FlatAdam)
    _train_steps(sp, opt, 3, visible=mode == "flat-visible")
    keep = torch.rand(4000, generator=torch.Generator().manual_seed(3)).lt(0.6).to(cuda)
    old = sp._mcmc_params()
    grouped = [p for grp in opt.param_groups for p in grp["params"]]          # the optimizer's own order
    if mode == "torch":
        before = {i: {k: t.clone() for k, t in opt.state[p].items()} for i, p in enumerate(old)}
    else:
        m, vv, starts, widths = opt.live_moments(old)
        before = {i: (m[s:s + p.numel()].view(p.shape).clone(), vv[s:s + p.numel()].view(p.shape).clone())
                  for i, (p, s) in enumerate(zip(old, starts))}
        step = opt.step_count
    sp.prune(keep, opt)
    new = sp._mcmc_params()
    k = keep
    if mode == "torch":
        for i, p in enumerate(new):
            st = opt.state[p]
            assert torch.equal(st["exp_avg"], before[i]["exp_avg"][k])
            assert torch.equal(st["exp_avg_sq"], before[i]["exp_avg_sq"][k])
            assert torch.equal(st["step"], before[i]["step"])
        assert all(any(p is q for q in grp["params"]) for grp in opt.param_groups for p in grp["params"])
        return
    for j, p in enumerate(grouped):
        i = next(i for i, q in enumerate(old) if q is p)
        sm, sv = opt._staged[j]
        assert torch.equal(sm, before[i][0][k]) and torch.equal(sv, before[i][1][k])
    if mode == "flat-visible":                                  # placed by the next step: unseen rows keep their bits
        opt.zero_grad(set_to_none=True)
        img = sp(0)
        (img - 0.5).abs().mean().backward()
        vis = sp.visible_mask().clone()
        opt.step(visible=vis)
        assert opt.step_count == step + 1
        m, vv, starts, _ = opt.live_moments(new)
        hidden = vis == 0
        assert bool(hidden.any())
        for i, (p, s) in enumerate(zip(new, starts)):
            got = m[s:s + p.numel()].view(p.shape)
            assert torch.equal(got[hidden], before[i][0][k][hidden])


def test_train_dp_prunes_to_half(gs, cuda):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_dp.py"), "--gaussians", "20000", "--res",
                        "160x120", "--iters", "150", "--views", "4", "--prune-at", "100", "--prune-keep", "0.5"],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "10000 Gaussians" in r.stdout.splitlines()[-1], r.stdout
