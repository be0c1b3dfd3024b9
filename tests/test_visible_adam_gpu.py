"""Visible-only Adam on the device: gs_adam_step_visible against the dense kernel (bit for bit on the visible rows,
untouched bits everywhere else) and against the CPU oracle of tests/visible_adam_oracle.py; gs_frame_visible against
the fp64 oracle's binning and the densification statistics' count; and a training run through
`FlatAdam.step(visible=Splatter.visible_mask())` with a densification and a checkpoint in the middle."""
import pytest
import torch

import synthetic as S
import visible_adam_oracle as VO
from test_densify_stats_gpu import CASES, NAMES, _device_frame, _oracle_stats, _splatter, _views

pytestmark = pytest.mark.gpu

BETAS, EPS = (0.9, 0.99), 1e-8
LRS = (0.003, 0.03, 0.05, 0.004, 0.005)


def _widths(d):
    return (3, d, 1, 4, 3)            # pos, rgb, opa, quat, scale: the order of renderer._flat_grads


def _state(n, d, dev, seed=0):
    """Flat buffers in the bucket's layout: random parameters, zero moments; plus a gradient maker (pads zero, as
    renderer._flat_grads leaves them)."""
    widths = _widths(d)
    starts, total = VO.layout(n, widths)
    gen = torch.Generator().manual_seed(seed)
    p = torch.randn(total, generator=gen).to(dev)
    elem = torch.zeros(total, dtype=torch.bool)
    for s0, w in zip(starts, widths):
        elem[s0:s0 + n * w] = True

    def grad(scale=1.0):
        return (torch.randn(total, generator=gen) * scale * elem).to(dev)

    ends = starts[1:] + [total]
    return dict(n=n, widths=widths, starts=starts, ends=ends, total=total, p=p, m=torch.zeros_like(p),
                v=torch.zeros_like(p), grad=grad, gen=gen)


def _dense(gaussian, st, p, m, v, g, step):
    gaussian.adam_step(p, g, m, v, st["ends"], list(LRS), *BETAS, EPS, step)


def _visible(gaussian, st, p, m, v, g, vis, step):
    gaussian.adam_step_visible(p, g, m, v, st["starts"], list(st["widths"]), list(LRS), vis, *BETAS, EPS, step)


def _row_elements(st, vis):
    """bool [total]: the floats of the visible rows of every segment."""
    out = torch.zeros(st["total"], dtype=torch.bool, device=vis.device)
    for s0, w in zip(st["starts"], st["widths"]):
        out[s0:s0 + st["n"] * w].view(st["n"], w)[vis.bool()] = True
    return out


def _mask(kind, n, f, gen, dev):
    if f == 0:
        return torch.zeros(n, dtype=torch.uint8, device=dev)
    if kind == "random":
        return (torch.rand(n, generator=gen) < f).to(torch.uint8).to(dev)
    run = 40                                                     # runs that straddle the 32-row groups
    on = torch.rand((n + run - 1) // run, generator=gen) < f
    return on.repeat_interleave(run)[:n].to(torch.uint8).to(dev)


@pytest.mark.parametrize("d", [3, 27, 48])
@pytest.mark.parametrize("n", [1, 31, 32, 33, 1000, 100003])
def test_all_visible_is_the_dense_kernel_bit_for_bit(gs, cuda, d, n):
    gaussian = gs[0]
    st = _state(n, d, cuda, seed=n + d)
    a = [st[k].clone() for k in "pmv"]
    b = [st[k].clone() for k in "pmv"]
    ones = torch.ones(n, dtype=torch.uint8, device=cuda)
    for step in range(1, 6):
        g = st["grad"](0.1 * step)
        _dense(gaussian, st, *a, g, step)
        _visible(gaussian, st, *b, g, ones, step)
    for x, y, name in zip(a, b, "pmv"):
        assert torch.equal(x, y), (name, int((x != y).sum()))


@pytest.mark.parametrize("kind", ["random", "runs"])
@pytest.mark.parametrize("f", [0.0, 0.1, 0.5])
@pytest.mark.parametrize("d", [3, 27, 48])
def test_masked_rows_match_dense_and_the_rest_is_untouched(gs, cuda, d, f, kind):
    gaussian = gs[0]
    n = 20011
    st = _state(n, d, cuda, seed=7)
    cur = [st[k] for k in "pmv"]
    for step in (1, 2):                                          # moments away from zero
        _dense(gaussian, st, *cur, st["grad"](), step)
    # pads included: give them values a stray write would change
    pad = ~_row_elements(st, torch.ones(n, dtype=torch.uint8, device=cuda))
    for t in cur:
        t[pad] = 3.25
    before = [t.clone() for t in cur]
    dense = [t.clone() for t in cur]
    vis = _mask(kind, n, f, st["gen"], cuda)
    g = st["grad"]()
    launches = gaussian.kernel_launches()
    _visible(gaussian, st, *cur, g, vis, 3)
    assert gaussian.kernel_launches() == launches + 1
    _dense(gaussian, st, *dense, g, 3)
    rows = _row_elements(st, vis)
    assert int(rows.sum()) == int(vis.sum()) * sum(st["widths"])
    for got, want, old, name in zip(cur, dense, before, "pmv"):
        assert torch.equal(got[rows], want[rows]), name
        assert torch.equal(got[~rows], old[~rows]), name
    if f == 0:
        assert all(torch.equal(x, y) for x, y in zip(cur, before))


def test_against_the_cpu_oracle(gs, cuda):
    gaussian = gs[0]
    n = 5003
    st = _state(n, 27, cuda, seed=3)
    dev = [st[k] for k in "pmv"]
    cpu = [t.cpu().clone() for t in dev]
    for step in range(1, 7):
        vis = _mask("random", n, 0.4, st["gen"], cuda)
        g = st["grad"](0.3 * step)
        _visible(gaussian, st, *dev, g, vis, step)
        VO.adam_visible(cpu[0], g.cpu(), cpu[1], cpu[2], st["starts"], st["widths"], LRS, n, vis.cpu(), *BETAS, EPS,
                        step)
    for got, want, name in zip(dev, cpu, "pmv"):
        err = float((got.cpu() - want).abs().max())
        assert err <= 1e-6 * float(want.abs().max()), (name, err)


def test_two_runs_give_the_same_bits(gs, cuda):
    gaussian = gs[0]
    outs = []
    for _ in range(2):
        st = _state(30011, 48, cuda, seed=11)
        cur = [st[k] for k in "pmv"]
        for step in range(1, 5):
            _visible(gaussian, st, *cur, st["grad"](), _mask("random", st["n"], 0.3, st["gen"], cuda), step)
        outs.append(cur)
    assert all(torch.equal(x, y) for x, y in zip(*outs))


@pytest.mark.parametrize("case", ["rgb", "sh27-gauss", "sh27-pixel", "rgb-dilate", "rgb-antialias", "rgb-packed"])
def test_frame_visible_is_the_oracles_binning(gs, cuda, case):
    """Per view: the mask equals count > 0 of the fp64 oracle's binning and the increment DensifyStats.count received
    from the same backward, and every Gaussian with a non-zero gradient row is in it."""
    sh_dim, sh_eval, mode, maps, packed, _ = CASES[case]
    n, w, h = (4000, 128, 96) if sh_dim == 3 or sh_eval == "gaussian" else (2500, 112, 80)
    g = S.make_gaussians(n, w, h, 0, sh_dim, (0.05, 0.9), (0.6, 5.0))
    g["pos"][::3] *= 3.0                                          # a third spread out: many of them off screen
    views = _views(w, h, 2)
    if packed:
        gs[0].tune("gather", 0)
    try:
        sp = _splatter(g, views, cuda, sh_eval=sh_eval, filter2d=mode, densify_stats="grad")
        masks, losses = [], []
        for j, v in enumerate(views):
            count0 = sp.densify_stats.count.clone()
            losses.append(_device_frame(sp, v, j, True, maps, 10 * j))
            mask = sp.visible_mask().clone()
            assert mask.dtype == torch.uint8 and mask.shape == (n,)
            assert torch.equal(mask.int(), sp.densify_stats.count - count0)
            touched = torch.zeros(n, dtype=torch.bool, device=cuda)
            for q in NAMES:
                gr = getattr(sp.gaussian_3ds, q).grad
                touched |= (gr.reshape(n, -1) != 0).any(1)
                getattr(sp.gaussian_3ds, q).grad = None
            assert not bool((touched & (mask == 0)).any())
            masks.append(mask.cpu())
        torch.cuda.synchronize()
    finally:
        gs[0].tune("gather", 1)
    assert 0 < int(masks[0].sum()) < n
    for j, v in enumerate(views):
        ref = _oracle_stats(g, [v], [losses[j]], sh_eval, mode, maps, False, cuda)
        assert torch.equal(masks[j].long(), (ref["count"] > 0).long()), j


def test_batch_mask_is_the_or_of_its_views_and_accumulate_ors(gs, cuda):
    g = S.make_gaussians(5000, 128, 96, 2, 27, (0.05, 0.9), (0.6, 5.0))
    sp = _splatter(g, _views(128, 96, 3), cuda, sh_eval="gaussian")
    singles = []
    with torch.no_grad():
        for j in range(3):
            sp(j)
            singles.append(sp.visible_mask().clone())
        union = singles[0] | singles[1] | singles[2]
        assert any(not torch.equal(s, union) for s in singles)
        sp.render_batch([0, 1, 2])
        assert torch.equal(sp.visible_mask(), union)
        sp(0)
        sp.visible_mask()
        sp(1)
        assert torch.equal(sp.visible_mask(accumulate=True), singles[0] | singles[1])
        o = sp.render_maps(2)
        assert torch.equal(sp.visible_mask(), singles[2]) and o["image"].shape[-1] == 3


def test_frame_visible_refusals_on_a_live_context(gs, cuda):
    gaussian = gs[0]
    mask = torch.zeros(100, dtype=torch.uint8, device=cuda)
    with pytest.raises(RuntimeError, match="no forward"):
        gaussian.RenderContext().visible_into(mask)
    g = S.make_gaussians(300, 64, 48, 0)
    sp = _splatter(g, _views(64, 48, 1), cuda)
    with torch.no_grad():
        sp(0)
    launches = gaussian.kernel_launches()
    with pytest.raises(RuntimeError, match="n differs"):
        sp._rctx.visible_into(mask)
    with pytest.raises(RuntimeError, match="uint8"):
        sp._rctx.visible_into(torch.zeros(300, device=cuda))
    assert gaussian.kernel_launches() == launches
    sp._rctx.visible_into(torch.zeros(300, dtype=torch.uint8, device=cuda))
    assert gaussian.kernel_launches() == launches + 1


def test_flat_adam_visible_argument_checks(gs, cuda):
    import optim
    import renderer
    n = 64
    ps = [torch.nn.Parameter(torch.randn(s, device=cuda)) for s in ((n, 3), (n, 3), (n,), (n, 4), (n, 3))]
    grads, _ = renderer._flat_grads(tuple(ps))
    for p, gv in zip(ps, grads):
        p.grad = gv.normal_()
    opt = optim.FlatAdam(ps, lr=0.01)
    with pytest.raises(ValueError, match="shape\\[0\\]"):
        opt.step(visible=torch.ones(n + 1, dtype=torch.uint8, device=cuda))
    with pytest.raises(TypeError):
        opt.step(visible=torch.ones(n, dtype=torch.bool, device=cuda))
    assert opt.step_count == 0
    before = [p.detach().clone() for p in ps]
    vis = torch.zeros(n, dtype=torch.uint8, device=cuda)
    vis[5] = 1
    opt.step(visible=vis)
    assert opt.step_count == 1
    for p, b in zip(ps, before):
        changed = (p.detach() != b).reshape(n, -1).any(1)
        assert bool(changed[5]) and int(changed.sum()) == 1


FAR = (10.0, 0.0, -10.0)      # behind the cameras of views 0, 1 and 2 (make_view: p_c.z = -s x + c z + 4 < 0)


def _student(n, w, h):
    teacher = S.make_gaussians(n, w, h, 0)
    gen = torch.Generator().manual_seed(100)
    st = {k: t.clone() for k, t in teacher.items()}
    st["pos"] += torch.randn(n, 3, generator=gen) * 0.01
    st["rgb"] = torch.zeros_like(teacher["rgb"])
    st["opa"] = torch.full_like(teacher["opa"], -2.0)
    for k in st:                                                  # one more Gaussian that no view ever bins
        st[k] = torch.cat([st[k], st[k][:1]])
    st["pos"][n] = torch.tensor(FAR)
    return teacher, st


def _make_opt(sp):
    import optim
    g = sp.gaussian_3ds
    return optim.FlatAdam([{"params": g.opa, "lr": 0.03}, {"params": g.rgb, "lr": 0.03}, {"params": g.pos, "lr": 0.003},
                           {"params": g.scale, "lr": 0.003}, {"params": g.quat, "lr": 0.003}], betas=BETAS)


def _train(sp, opt, gts, first, steps, hist=None):
    for it in range(first, first + steps):
        j = it % len(gts)
        opt.zero_grad()
        loss = (sp(j) - gts[j]).abs().mean()
        loss.backward()
        opt.step(visible=sp.visible_mask())
        if hist is not None:
            hist.append(float(loss.detach()))


def _far_row(sp, opt):
    """(parameters, moments) of the Gaussian at FAR, wherever the densification moved it."""
    g = sp.gaussian_3ds
    i = (g.pos.detach() == torch.tensor(FAR, device=g.pos.device)).all(1).nonzero()
    assert i.numel() == 1
    i = int(i)
    params = torch.cat([getattr(g, q).detach()[i].reshape(-1) for q in NAMES])
    flat, m, v, ordered, _, base = opt._flat
    mom = []
    for p in ordered:
        o, w = p.grad.storage_offset() - base, p.numel() // p.shape[0]
        mom += [m[o + i * w:o + (i + 1) * w], v[o + i * w:o + (i + 1) * w]]
    return params.clone(), torch.cat(mom).clone()


def test_training_with_visible_adam_densification_and_resume(gs, cuda, tmp_path):
    """60 steps on the synthetic multi-view scene: the loss falls as in the dense loop's test
    (test_frame_gpu.test_training_loop_converges: below 0.6 of the start); the Gaussian no camera sees keeps its
    parameters bit for bit and its moments at zero; a densification in the middle re-sizes the mask; and a checkpoint
    taken mid-run resumes bit-exactly."""
    import checkpoint
    n, w, h = 20000, 160, 96
    teacher, student = _student(n, w, h)
    views = _views(w, h, 3)
    with torch.no_grad():
        tsp = _splatter(teacher, views, cuda)
        gts = [tsp(j).clone() for j in range(3)]
    sp = _splatter(student, views, cuda, densify_stats="grad")
    opt = _make_opt(sp)
    hist = []
    _train(sp, opt, gts, 0, 30, hist)
    assert sp.visible_mask().numel() == n + 1 and 0 < int(sp.visible_mask().sum()) <= n
    far0 = torch.cat([student[q][n].reshape(-1) for q in NAMES]).to(cuda)
    params, mom = _far_row(sp, opt)
    assert torch.equal(params, far0) and not bool(mom.any())

    info = sp.adaptive_control_screen(0.01, 10.0, grad_thresh=2e-4)
    assert info["total"] != n + 1
    opt = _make_opt(sp)                                           # the parameters are new: so is the optimizer
    _train(sp, opt, gts, 30, 10, hist)
    assert sp.visible_mask().numel() == info["total"]
    path = str(tmp_path / "ckpt.pth")
    sp.save_checkpoint(path, optimizer=opt, iteration=40)
    _train(sp, opt, gts, 40, 5, hist)
    want = {q: getattr(sp.gaussian_3ds, q).detach().clone() for q in NAMES}
    want_m = [t.clone() for t in opt._flat[1:3]]

    sp2 = _splatter(student, views, cuda, densify_stats="grad")
    checkpoint.load_checkpoint(path, sp2, None)
    opt2 = _make_opt(sp2)
    checkpoint.load_checkpoint(path, None, opt2)
    _train(sp2, opt2, gts, 40, 5)
    assert opt2.step_count == opt.step_count == 15
    for q in NAMES:
        assert torch.equal(getattr(sp2.gaussian_3ds, q).detach(), want[q]), q
    for a, b in zip(opt2._flat[1:3], want_m):
        assert torch.equal(a, b)

    _train(sp, opt, gts, 45, 15, hist)
    assert len(hist) == 60
    first, last = sum(hist[:3]) / 3, sum(hist[-3:]) / 3
    assert last < 0.6 * first, (first, last)
    params, mom = _far_row(sp, opt)
    assert torch.equal(params, far0) and not bool(mom.any())
