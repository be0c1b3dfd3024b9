"""MCMC densification on the device against the fp64 oracle of tests/mcmc_oracle.py: the sampler draw by draw,
relocation and growth row by row (new opacity / scale to 1e-6, copies and untouched floats bit for bit, moments zeroed
exactly where they must be), the position noise, the optimizer state across a growth (FlatAdam and torch.optim.Adam,
checkpoints included), and a short MCMC training run that is reproducible and resumable bit for bit."""
import numpy as np
import pytest
import torch

import mcmc_oracle as MO
import synthetic as S
import visible_adam_oracle as VO
from test_densify_stats_gpu import _splatter, _views

pytestmark = pytest.mark.gpu

ACT = {"abs": 0, "exp": 1}
KEYS = ("pos", "rgb", "opa", "quat", "scale", "feat")


def _params(n, d, act, f=0, dead=0.1, seed=0):
    """float32 numpy parameters: 1-in-10 dead (sigmoid(-7) < 0.005), pos[:, 0] = the row index (a row's origin is
    readable from any copy), raw scales of 0.01 .. 0.3 in either sign (abs) or their logs (exp)."""
    rng = np.random.default_rng(seed)
    pos = rng.normal(size=(n, 3)).astype(np.float32)
    pos[:, 0] = np.arange(n)
    opa = rng.normal(0.0, 2.0, size=n).astype(np.float32)
    opa[rng.random(n) < dead] = -7.0
    s = rng.uniform(0.01, 0.3, size=(n, 3))
    scale = (np.where(rng.random((n, 3)) < 0.5, -s, s) if act == "abs" else np.log(s)).astype(np.float32)
    return dict(pos=pos, rgb=rng.normal(size=(n, d)).astype(np.float32), opa=opa,
                quat=rng.normal(size=(n, 4)).astype(np.float32), scale=scale,
                feat=rng.normal(size=(n, f)).astype(np.float32) if f else None)


def _dev(p, cuda):
    return {k: (None if a is None else torch.from_numpy(a.copy()).to(cuda)) for k, a in p.items()}


def _host(p):
    return {k: (None if a is None else a.cpu().numpy()) for k, a in p.items()}


def _close(got, want, rel=1e-6, atol=1e-6):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return bool((np.abs(got - want) <= rel * np.abs(want) + atol).all())


def _check_rows(got, want, rows):
    """Rows `rows` (bool): opa and scale to 1e-6 of the oracle, every other parameter bit-exact; the other rows bit
    for bit what the oracle (= the input) has."""
    for k in KEYS:
        if want[k] is None:
            continue
        g, w = got[k], want[k]
        if k in ("opa", "scale"):
            assert _close(g[rows], w[rows]), k
            assert np.array_equal(g[~rows], w[~rows]), k
        else:
            assert np.array_equal(g, w), k


def _grow(gaussian, d, u, cuda):
    return gaussian.mcmc_add(d["pos"], d["rgb"], d["opa"], d["quat"], d["scale"], None, 1, 0.005,
                             torch.from_numpy(u).to(cuda))


def test_sampler_matches_the_oracle_draw_by_draw(gs, cuda):
    """The prefix sums are integers, so the draws are the oracle's exactly; the only allowance is for a weight whose
    o 2^32 the device's fp64 sigmoid rounds the other way (near, asserted absent for these seeds)."""
    gaussian = gs[0]
    for seed, n, n_new in ((0, 1000, 700), (1, 50021, 3000), (2, 2_400_000, 120_000)):
        p = _params(n, 3, "exp", seed=seed)
        p["opa"][::7] = -30.0                                   # runs of zero weight (o 2^32 rounds to 0)
        p["opa"][3::11] = -20.0                                 # tiny weights: o 2^32 ~ 9
        u = np.random.default_rng(seed + 10).random(n_new).astype(np.float32)
        src, near = MO.sample(MO.weights(MO.sigmoid(p["opa"])), u)
        assert int(near.sum()) == 0, int(near.sum())
        d = _dev(p, cuda)
        out = _grow(gaussian, d, u, cuda)
        got = out[0][n:, 0].cpu().numpy().astype(np.int64)          # pos[:, 0] is the source's index
        assert np.array_equal(got, src)
        if n_new > 10_000:                                            # C3 size: same inputs, same bits
            again = _grow(gaussian, d, u, cuda)
            assert all(torch.equal(a, b) for a, b in zip(out, again))
            continue
        want, _, _ = MO.add(p, "exp", 0.005, u)                     # counts enter through the new opacity / scale
        rows = np.zeros(n + n_new, dtype=bool)
        rows[src] = True
        rows[n:] = True
        _check_rows(_host(dict(zip(KEYS, out + [None]))), want, rows)


def test_growth_with_no_weight_appends_plain_copies_of_row_0(gs, cuda):
    gaussian = gs[0]
    p = _params(100, 3, "abs")
    p["opa"][:] = -40.0                                         # every o 2^32 rounds to 0
    d = _dev(p, cuda)
    out = _host(dict(zip(KEYS, _grow(gaussian, d, np.random.default_rng(0).random(7).astype(np.float32), cuda)
                         + [None])))
    want, _, _ = MO.add(p, "abs", 0.005, np.zeros(7, dtype=np.float32))
    for k in KEYS[:5]:
        assert np.array_equal(out[k], want[k]), k
        assert np.array_equal(out[k][:100], p[k]), k


def _moments(n, widths, cuda, seed):
    starts, total = VO.layout(n, widths)
    gen = torch.Generator().manual_seed(seed)
    m = torch.randn(total, generator=gen).to(cuda)
    v = torch.rand(total, generator=gen).to(cuda)
    return m, v, starts


def _moment_rows(t, starts, widths, n):
    return [t[s:s + n * w].view(n, w) for s, w in zip(starts, widths)]


@pytest.mark.parametrize("f", [0, 8])
@pytest.mark.parametrize("act", ["abs", "exp"])
@pytest.mark.parametrize("d", [3, 48])
def test_relocation_matches_the_oracle(gs, cuda, d, act, f):
    gaussian = gs[0]
    n = 20011
    p = _params(n, d, act, f, seed=d + f)
    u = np.random.default_rng(3).random(n).astype(np.float32)
    want, touched, k, near = MO.relocate(p, act, 0.005, u)
    assert k > 1000 and int(near.sum()) == 0
    dv = _dev(p, cuda)
    widths = [3, d, 1, 4, 3]                                        # pos, rgb, opa, quat, scale
    m, v, starts = _moments(n, widths, cuda, seed=d)
    m0, v0 = m.clone(), v.clone()
    mask = torch.zeros(n, dtype=torch.uint8, device=cuda)
    n_rel = gaussian.mcmc_relocate(dv["pos"], dv["rgb"], dv["opa"], dv["quat"], dv["scale"], dv["feat"], ACT[act],
                                   0.005, torch.from_numpy(u).to(cuda), exp_avg=m, exp_avg_sq=v, seg_starts=starts,
                                   seg_widths=widths, touched=mask)
    assert n_rel.is_cuda and int(n_rel) == k
    assert np.array_equal(mask.cpu().numpy().astype(bool), touched)
    _check_rows(_host(dv), want, touched)
    rows = torch.from_numpy(touched).to(cuda)
    for t, t0 in ((m, m0), (v, v0)):
        expect = t0.clone()
        for seg in _moment_rows(expect, starts, widths, n):
            seg[rows] = 0.0
        assert torch.equal(t, expect)                               # pads and untouched rows included


def test_relocation_edge_cases(gs, cuda):
    gaussian = gs[0]

    def run(p, act="abs"):
        dv = _dev(p, cuda)
        n = len(p["opa"])
        u = np.random.default_rng(9).random(n).astype(np.float32)
        n_rel = gaussian.mcmc_relocate(dv["pos"], dv["rgb"], dv["opa"], dv["quat"], dv["scale"], None, ACT[act], 0.005,
                                       torch.from_numpy(u).to(cuda))
        want, touched, k, _ = MO.relocate(p, act, 0.005, u)
        assert int(n_rel) == k
        return _host(dv), want, touched, k

    p = _params(500, 3, "abs", dead=0.0)                              # nothing dead: no bit changes
    p["opa"] = np.abs(p["opa"])
    got, _, _, k = run(p)
    assert k == 0 and all(np.array_equal(got[q], p[q]) for q in KEYS[:5])
    p = _params(300, 3, "abs", dead=1.0)                              # everything dead: a no-op
    got, _, _, k = run(p)
    assert k == 0 and all(np.array_equal(got[q], p[q]) for q in KEYS[:5])
    p = _params(61, 3, "abs", dead=1.0)                               # one alive and 60 dead: r clamps at 51
    p["opa"][17] = 2.0
    got, want, touched, k = run(p)
    assert k == 60 and touched.all()
    _check_rows(got, want, touched)
    o51, _, _ = MO.ratio(float(MO.sigmoid(2.0)), 51)
    assert abs(MO.sigmoid(got["opa"][17]) - max(o51, 0.005)) < 1e-6
    assert (got["pos"][:, 0] == 17).all()
    for dead in (0.0, 1.0):                                           # n = 1
        p = _params(1, 3, "exp", dead=dead)
        got, _, _, k = run(p, "exp")
        assert k == 0 and all(np.array_equal(got[q], p[q]) for q in KEYS[:5])


def _student(n, w, h, seed=100):
    teacher = S.make_gaussians(n, w, h, 0)
    gen = torch.Generator().manual_seed(seed)
    st = {k: t.clone() for k, t in teacher.items()}
    st["pos"] += torch.randn(n, 3, generator=gen) * 0.02
    st["rgb"] = torch.zeros_like(teacher["rgb"])
    st["opa"] = torch.randn(n, generator=gen) * 2.0
    st["opa"][::8] = -7.0                                             # dead from the start
    return teacher, st


def _make_opt(sp, kind="flat"):
    import optim
    g = sp.gaussian_3ds
    groups = [{"params": [g.opa], "lr": 0.03}, {"params": [g.rgb], "lr": 0.03}, {"params": [g.pos], "lr": 0.001},
              {"params": [g.scale], "lr": 0.003}, {"params": [g.quat], "lr": 0.003}]
    if kind == "flat":
        return optim.FlatAdam(groups, betas=(0.9, 0.99))
    return torch.optim.Adam(groups, betas=(0.9, 0.99), eps=1e-8)


def _scene(cuda, n=3000, w=160, h=96):
    teacher, student = _student(n, w, h)
    views = _views(w, h, 3)
    with torch.no_grad():
        tsp = _splatter(teacher, views, cuda)
        gts = [tsp(j).clone() for j in range(3)]
    return student, views, gts


def _step(sp, opt, gts, it, mc=None):
    j = it % len(gts)
    opt.zero_grad()
    loss = (sp(j) - gts[j]).abs().mean()
    loss.backward()
    if mc is not None:
        mc.after_backward(it)
    opt.step()
    return float(loss.detach())


NAMES = ("pos", "rgb", "opa", "quat", "scale")


def _moments_of(opt, sp):
    """{name: (exp_avg [n, w], exp_avg_sq [n, w])} of either optimizer."""
    g = sp.gaussian_3ds
    out = {}
    if hasattr(opt, "live_moments"):
        m, v, starts, widths = opt.live_moments([getattr(g, q) for q in NAMES])
        _, _, _, ordered, _, _ = opt._flat
        for p, s, w in zip(ordered, starts, widths):
            q = next(q for q in NAMES if getattr(g, q) is p)
            out[q] = (m[s:s + p.numel()].view(p.shape[0], -1).clone(), v[s:s + p.numel()].view(p.shape[0], -1).clone())
    else:
        for q in NAMES:
            st = opt.state[getattr(g, q)]
            out[q] = (st["exp_avg"].view(st["exp_avg"].shape[0], -1).clone(),
                      st["exp_avg_sq"].view(st["exp_avg"].shape[0], -1).clone())
    return out


@pytest.mark.parametrize("kind", ["flat", "torch"])
def test_splatter_relocation_zeroes_exactly_the_touched_moment_rows(gs, cuda, kind):
    student, views, gts = _scene(cuda)
    sp = _splatter(student, views, cuda)
    opt = _make_opt(sp, kind)
    for it in range(3):
        _step(sp, opt, gts, it)
    g = sp.gaussian_3ds
    ids = [id(getattr(g, q)) for q in NAMES]
    before = {q: getattr(g, q).detach().cpu().numpy().copy() for q in NAMES}
    mom0 = _moments_of(opt, sp)
    n = g.pos.shape[0]
    p = dict(before, feat=None)
    gen = torch.Generator(device=cuda).manual_seed(5)
    u = torch.rand(n, device=cuda, generator=torch.Generator(device=cuda).manual_seed(5)).cpu().numpy()
    want, touched, k, near = MO.relocate(p, "abs", 0.005, u)
    assert k > 100 and int(near.sum()) == 0
    n_rel = sp.mcmc_relocate(opt, generator=gen)
    assert int(n_rel) == k and [id(getattr(g, q)) for q in NAMES] == ids
    _check_rows(_host({q: getattr(g, q).detach() for q in NAMES} | {"feat": None}), want, touched)
    mom1 = _moments_of(opt, sp)
    rows = torch.from_numpy(touched).to(cuda)
    for q in NAMES:
        for a, b in zip(mom1[q], mom0[q]):
            assert torch.equal(a[~rows], b[~rows]), q
            assert not bool(a[rows].any()), q
            assert torch.equal(torch.signbit(a[rows]), torch.zeros_like(a[rows], dtype=torch.bool)), q
    _step(sp, opt, gts, 3)                                            # the optimizer still runs on the same Parameters


@pytest.mark.parametrize("kind", ["flat", "torch"])
def test_growth_keeps_the_moments_and_the_next_step_is_dense_adam(gs, cuda, kind):
    gaussian = gs[0]
    student, views, gts = _scene(cuda)
    sp = _splatter(student, views, cuda, densify_stats="grad")
    opt = _make_opt(sp, kind)
    for it in range(3):
        _step(sp, opt, gts, it)
    n = sp.gaussian_3ds.pos.shape[0]
    assert sp.mcmc_add(n, optimizer=opt) == 0                         # at the cap: a no-op
    assert sp.mcmc_add(n + 10 ** 6, growth=1.0, optimizer=opt) == 0
    mom0 = _moments_of(opt, sp)
    added = sp.mcmc_add(int(1.2 * n), optimizer=opt)                  # below the cap: int(1.05 n) - n
    assert added == int(1.05 * n) - n and sp.n_gaussians == n + added == sp.gaussian_3ds.pos.shape[0]
    g = sp.gaussian_3ds
    j = 3 % len(gts)
    opt.zero_grad()
    (sp(j) - gts[j]).abs().mean().backward()
    assert sp.densify_stats.n == n + added
    before = {q: getattr(g, q).detach().clone() for q in NAMES}
    grads = {q: getattr(g, q).grad.clone() for q in NAMES}
    step0 = opt.step_count if kind == "flat" else int(opt.state[g.pos]["step"])
    opt.step()
    mom1 = _moments_of(opt, sp)
    lrs = {"opa": 0.03, "rgb": 0.03, "pos": 0.001, "scale": 0.003, "quat": 0.003}
    for q in NAMES:                                                   # dense Adam on the carried / zero moments
        pf = before[q].reshape(-1).clone()
        pf = torch.cat([pf, pf.new_zeros((-pf.numel()) % 4)])
        gf = torch.cat([grads[q].reshape(-1), pf.new_zeros((-grads[q].numel()) % 4)])
        mf, vf = (torch.cat([mom0[q][i].reshape(-1), pf.new_zeros(pf.numel() - mom0[q][i].numel())]) for i in (0, 1))
        if kind == "flat":
            gaussian.adam_step(pf, gf, mf, vf, [pf.numel()], [lrs[q]], 0.9, 0.99, 1e-8, step0 + 1)
            assert torch.equal(getattr(g, q).detach().reshape(-1), pf[:before[q].numel()]), q
            assert torch.equal(mom1[q][0].reshape(-1), mf[:before[q].numel()]), q
            assert torch.equal(mom1[q][1].reshape(-1), vf[:before[q].numel()]), q
        else:
            ref = torch.nn.Parameter(before[q].clone())
            ref.grad = grads[q]
            ro = torch.optim.Adam([ref], lr=lrs[q], betas=(0.9, 0.99), eps=1e-8)
            ro.state[ref] = {"step": torch.tensor(float(step0)), "exp_avg": mf[:ref.numel()].view(ref.shape).clone(),
                             "exp_avg_sq": vf[:ref.numel()].view(ref.shape).clone()}
            ro.step()
            assert torch.equal(getattr(g, q).detach(), ref.detach()), q


def test_checkpoint_between_growth_and_step_resumes_bit_exactly(gs, cuda, tmp_path):
    import checkpoint
    student, views, gts = _scene(cuda)
    sp = _splatter(student, views, cuda)
    opt = _make_opt(sp)
    for it in range(4):
        _step(sp, opt, gts, it)
    sp.mcmc_add(10 ** 6, optimizer=opt)
    path = str(tmp_path / "ckpt.pth")
    sp.save_checkpoint(path, optimizer=opt, iteration=4)
    for it in range(4, 8):
        _step(sp, opt, gts, it)
    want = {q: getattr(sp.gaussian_3ds, q).detach().clone() for q in NAMES}
    want_m = [t.clone() for t in opt._flat[1:3]]
    sp2 = _splatter(student, views, cuda)
    checkpoint.load_checkpoint(path, sp2, None)
    opt2 = _make_opt(sp2)
    checkpoint.load_checkpoint(path, None, opt2)
    for it in range(4, 8):
        _step(sp2, opt2, gts, it)
    assert opt2.step_count == opt.step_count == 8
    for q in NAMES:
        assert torch.equal(getattr(sp2.gaussian_3ds, q).detach(), want[q]), q
    for a, b in zip(opt2._flat[1:3], want_m):
        assert torch.equal(a, b)


@pytest.mark.parametrize("act", ["abs", "exp"])
def test_noise_with_given_z_matches_the_oracle(gs, cuda, act):
    gaussian = gs[0]
    n = 100003
    p = _params(n, 3, act, seed=4)
    p["opa"] = np.random.default_rng(5).uniform(-9.0, 3.0, size=n).astype(np.float32)   # across the gate
    z = np.random.default_rng(6).normal(size=(n, 3)).astype(np.float32)
    dv = _dev(p, cuda)
    dv["pos"].zero_()                                                 # the new positions are the displacement
    keep = {q: dv[q].clone() for q in ("rgb", "opa", "quat", "scale")}
    gaussian.mcmc_noise(dv["pos"], dv["quat"], dv["scale"], dv["opa"], ACT[act], 0.75, 1, torch.from_numpy(z).to(cuda))
    want = MO.noise_delta(p["quat"], p["scale"], p["opa"], act, 0.75, z)
    got = dv["pos"].cpu().numpy().astype(np.float64)
    err = np.abs(got - want).max()
    assert err <= 1e-6 * np.abs(want).max(), err
    row = np.abs(got - want).max(1) / np.maximum(np.abs(want).max(1), 1e-30)
    assert np.median(row) < 1e-6
    for q, t in keep.items():
        assert torch.equal(dv[q], t), q


def test_noise_philox_is_deterministic_and_normal(gs, cuda):
    gaussian = gs[0]
    n = 2_400_000
    quat = torch.tensor([1.0, 0.0, 0.0, 0.0], device=cuda).repeat(n, 1)
    scale = torch.zeros(n, 3, device=cuda)                            # exp: s = 1, Sigma = I
    opa = torch.full((n,), -20.0, device=cuda)                        # a constant gate
    runs = []
    for seed in (12345, 12345, 54321):
        pos = torch.zeros(n, 3, device=cuda)
        gaussian.mcmc_noise(pos, quat, scale, opa, 1, 2.0, seed)
        runs.append(pos)
    assert torch.equal(runs[0], runs[1]) and not torch.equal(runs[0], runs[2])
    assert float((runs[0] != runs[2]).float().mean()) > 0.99
    g = float(MO.gate(np.array([-20.0]))[0])
    x = runs[0].double() / (2.0 * g)
    mean = x.mean(0)
    cov = torch.cov(x.T)
    tol = 5.0 / n ** 0.5                                              # 5 sigma of the sample mean
    assert float(mean.abs().max()) < tol, mean
    assert float((cov - torch.eye(3, device=cuda, dtype=torch.float64)).abs().max()) < 5.0 * (2.0 / n) ** 0.5, cov
    assert torch.equal(quat, torch.tensor([1.0, 0.0, 0.0, 0.0], device=cuda).repeat(n, 1))
    assert not bool(scale.any()) and bool((opa == -20.0).all())


def _mcmc_run(cuda, student, views, gts, iters, hist=None, ckpt=None, resume=None):
    """MCMC training (refine every 20 steps from step 50, cap 1.3 n0).  ckpt=(it, path) saves after step it - 1;
    resume=path continues from that checkpoint."""
    import checkpoint
    import mcmc
    n0 = student["pos"].shape[0]
    cap = int(1.3 * n0)
    torch.manual_seed(1234)
    sp = _splatter(student, views, cuda)
    first = 0
    if resume is not None:
        checkpoint.load_checkpoint(resume, sp, None)
    opt = _make_opt(sp)
    if resume is not None:
        first = checkpoint.load_checkpoint(resume, None, opt)["resume"]["iteration"]
    mc = mcmc.MCMC(sp, opt, cap, refine_start=50, refine_stop=10 ** 9, refine_every=20)
    for it in range(first, iters):
        if ckpt is not None and it == ckpt[0]:
            sp.save_checkpoint(ckpt[1], optimizer=opt, iteration=it)
        loss = _step(sp, opt, gts, it, mc)
        if hist is not None:
            hist.append(loss)
        g = sp.gaussian_3ds
        if mc.is_refine_step(it):
            dead = (torch.sigmoid(g.opa.detach().double()) <= float(np.float32(0.005))).cpu().numpy()
            rgb0 = g.rgb.detach().cpu().numpy()
            out = mc.after_step(it, 1e-4)
            rgb1 = g.rgb.detach().cpu().numpy()[:len(dead)]
            assert int(out["relocated"]) == int(dead.sum())
            alive = {r.tobytes() for r in rgb0[~dead]}                 # every dead one is now a copy of an alive one
            assert all(r.tobytes() in alive for r in rgb1[dead])
            assert np.array_equal(rgb1[~dead], rgb0[~dead])
        else:
            mc.after_step(it, 1e-4)
        assert sp.gaussian_3ds.pos.shape[0] <= cap
    return sp, opt


def test_mcmc_training_end_to_end(gs, cuda, tmp_path):
    student, views, gts = _scene(cuda)
    n0 = student["pos"].shape[0]
    hist = []
    path = str(tmp_path / "mid.pth")
    sp, opt = _mcmc_run(cuda, student, views, gts, 200, hist, ckpt=(110, path))
    assert sp.gaussian_3ds.pos.shape[0] == int(1.3 * n0)             # grown to the cap (by 5 % per refine step)
    first, last = sum(hist[:5]) / 5, sum(hist[-5:]) / 5
    assert last < 0.8 * first, (first, last)
    sp2, opt2 = _mcmc_run(cuda, student, views, gts, 200)
    sp3, opt3 = _mcmc_run(cuda, student, views, gts, 200, resume=path)
    for other, o in ((sp2, opt2), (sp3, opt3)):
        for q in NAMES:
            assert torch.equal(getattr(other.gaussian_3ds, q).detach(), getattr(sp.gaussian_3ds, q).detach()), q
        for a, b in zip(o._flat[1:3], opt._flat[1:3]):
            assert torch.equal(a, b)


def test_relocation_between_checkpoint_load_and_step_zeroes_the_restored_moments(gs, cuda, tmp_path):
    """A FlatAdam whose moments come from a checkpoint holds them outside a live flat buffer until its next step; a
    relocation in between must still zero the touched rows: the resumed run equals the uninterrupted one bit for bit."""
    import checkpoint
    student, views, gts = _scene(cuda)
    sp = _splatter(student, views, cuda)
    opt = _make_opt(sp)
    for it in range(3):
        _step(sp, opt, gts, it)
    path = str(tmp_path / "ckpt.pth")
    sp.save_checkpoint(path, optimizer=opt, iteration=3)
    sp2 = _splatter(student, views, cuda)
    checkpoint.load_checkpoint(path, sp2, None)
    opt2 = _make_opt(sp2)
    checkpoint.load_checkpoint(path, None, opt2, restore_rng=False)
    assert opt2._flat is None and opt2._resume[0] is not None
    for s, o in ((sp, opt), (sp2, opt2)):
        n_rel = s.mcmc_relocate(o, generator=torch.Generator(device=cuda).manual_seed(8))
        assert int(n_rel) > 100
        _step(s, o, gts, 3)
    assert opt2.step_count == opt.step_count == 4
    for q in NAMES:
        assert torch.equal(getattr(sp2.gaussian_3ds, q).detach(), getattr(sp.gaussian_3ds, q).detach()), q
    for a, b in zip(opt2._flat[1:3], opt._flat[1:3]):
        assert torch.equal(a, b)
