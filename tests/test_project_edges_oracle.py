"""CPU checks of tests/project_edges.py: the instantiation table against the two dispatches' literal mappings, each
scene's design (instance counts and live rows per run, n and the CTA layout, activation values, margins), and
the comparator's power (it fails on a dropped, duplicated or stale row, a non-zero row where the oracle's is zero
and a missing 3-D filter chain, and passes
an fp32 evaluation of the same oracle)."""
import functools
import os

import pytest
import torch

import project_edges as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def _scene(name):
    return P.BUILDERS[name]()


def test_table_matches_the_dispatch_sources():
    triples, tiers, stats_tiers = P.dispatch_literals(ROOT)
    rows = P.table()
    want = {(kg, d, gw) for (kg, d, gw), _ in P.COLOURS.values()}
    assert triples == want, (triples, want)
    assert sorted(tiers) == sorted(P.TIER_CODE.values()) and len(tiers) == len(P.TIERS)
    for kernel in ("bwd", "fwd", "bwd_batch", "fwd_batch"):
        assert {r["tier"] for r in rows if r["kernel"] == kernel} == set(P.TIERS), kernel
    bwd = {(r["kg"], r["d"], r["gw"]) for r in rows if r["kernel"] == "bwd"}
    assert bwd == want
    assert {r["kg"] for r in rows if r["kernel"] == "bwd_batch"} == {0, 9, 16}
    assert {r["kg"] for r in rows if r["kernel"] in ("fwd", "fwd_batch")} == {0, 9, 16}
    # the statistics: every tier of densify_stats_dispatch, with and without absgrad, single and batched
    code = {v: k for k, v in P.TIER_CODE.items()}
    for kernel in ("stats", "stats_batch"):
        got = {(r["tier"], r["absgrad"]) for r in rows if r["kernel"] == kernel}
        assert got == {(code[t], a) for t in stats_tiers for a in (False, True)}, kernel
    # every (DT, CG) pair of each colour family and tier; CG only with RGB rows
    for r in rows:
        if r["kernel"] == "bwd" and r["cg"]:
            assert r["kg"] > 0 or r["d"] == 3
    assert len({P.row_id(r) for r in rows}) == len(rows)


def test_table_fails_without_a_tier_line(tmp_path):
    """A scratch copy of project.cu with one by_tier case deleted no longer matches the table."""
    src = os.path.join(ROOT, "3d-gaussian-splatting_b200", "csrc")
    dst = tmp_path / "3d-gaussian-splatting_b200" / "csrc"
    dst.mkdir(parents=True)
    with open(os.path.join(src, "project.cu")) as f:
        text = f.read()
    line = "      case GS_TIER_FILT3D: return by_dt(kg, dd, gw, Int<GS_TIER_FILT3D>{});\n"
    assert line in text
    (dst / "project.cu").write_text(text.replace(line, ""))
    with open(os.path.join(src, "densify_stats.cu")) as f:
        (dst / "densify_stats.cu").write_text(f.read())
    _, tiers, _ = P.dispatch_literals(str(tmp_path))
    assert sorted(tiers) != sorted(P.TIER_CODE.values())


@pytest.mark.parametrize("name", ["frame-abs", "frame-exp"])
def test_frame_scene_hits_its_targets(name):
    sc = _scene(name)
    assert sc.n == P.N and sc.n % 32 == 1 and sc.n - 2 * 256 == 33
    fe = P.front(sc, 0, "none", None)
    counts = (fe["rects"][:, 1] - fe["rects"][:, 0]) * (fe["rects"][:, 3] - fe["rects"][:, 2])
    for run, (gid, rect, live) in sc.runs.items():
        assert tuple(fe["rects"][gid].tolist()) == rect, run
        rows = P.live_rows(sc, gid)
        assert [k for k, x in enumerate(rows) if x] == list(live), (run, rows)
    assert sorted(int(counts[gid]) for run, (gid, _, _) in sc.runs.items() if run.startswith("run")) == \
        [1, 2, 3, 4, 5, 7, 8, 9, 12, 13]
    # live and stale rows mixed inside one group of four, and a binned Gaussian hidden behind walls everywhere
    mixed = [run for run, (gid, _, live) in sc.runs.items()
             if 0 < len([k for k in live if k < 4]) < min(4, int(counts[gid]))]
    assert sorted(mixed) == ["siteA", "siteB", "siteC"], mixed
    hid = sc.runs["siteH"][0]
    assert int(counts[hid]) == 2 and sc.runs["siteH"][2] == ()
    ref = P.oracle(sc, "rgb", "none", None, False)["grads"]
    assert all(bool((g[hid] == 0).all()) for g in ref.values())
    roles = sc.roles
    unb = [i for i, r in enumerate(roles) if r == "unbinned"]
    assert all(bool(fe["mask"][i]) and int(counts[i]) == 0 for i in unb)
    # activation edges
    raw = sc.g["scale"]
    acts = [i for i, r in enumerate(roles) if r == "act"]
    assert set(raw[acts].abs().flatten().tolist()) == {0.5, 1.5}
    if sc.act == "abs":
        assert int((raw == 0).sum()) >= 10
    else:
        assert bool((raw[acts].abs() > 1).any()) and bool((raw[acts].abs() < 1).any())
    qn = sc.g["quat"].norm(dim=1)
    assert bool(((qn - 0.25).abs() < 1e-6).any()) and bool(((qn - 4).abs() < 1e-5).any())
    assert bool((sc.g["opa"] == 5.9).any()) and bool((sc.g["opa"] == -5.9).any())
    # 3-D filter: zero for some, comparable to the smallest activated scale for others
    s = raw.double().abs() + 1e-4 if sc.act == "abs" else raw.double().exp()
    on = sc.f3d > 0
    assert 50 < int(on.sum()) < sc.n - 50
    ratio = sc.f3d[on].double() / s[on].amin(1)
    assert float(ratio.min()) >= 0.49 and float(ratio.max()) <= 1.51
    assert not bool(P.unstable(sc).any())


@pytest.mark.parametrize("name", ["batch-abs", "batch-exp"])
def test_batch_scene_hits_its_targets(name):
    sc = _scene(name)
    assert sc.n == P.N and len(sc.views) == 3
    binned = []
    for v in range(3):
        fe = P.front(sc, v, "none", None)
        counts = (fe["rects"][:, 1] - fe["rects"][:, 0]) * (fe["rects"][:, 3] - fe["rects"][:, 2])
        binned.append(counts > 0)
        cta = [int((counts[k * 256:(k + 1) * 256] > 0).sum()) for k in range(3)]
        # view 0: rows in all three CTAs; views 1 and 2: none in the second CTA, rows in the first and third
        assert cta[0] > 0 and cta[2] > 0, (v, cta)
        assert (cta[1] > 0) == (v == 0), (v, cta)
    seen = torch.stack(binned).sum(0)
    assert int((seen == 1).sum()) >= 100 and int((seen == 3).sum()) >= 100     # some seen in one view only
    assert len({(vw.fx, tuple(vw.tran.tolist())) for vw in sc.views}) == 3
    assert not bool(P.unstable(sc).any())


def _row_contrib(sc, colour, tier, gid, t):
    """Gaussian gid's gradient from tile t alone (the row its instance there writes)."""
    r = P.oracle(sc, colour, tier, None, False, tiles=[t])
    return {q: g[gid] for q, g in r["grads"].items()}


def test_every_live_row_is_visible():
    """Each live row of each designed run moves its Gaussian's opacity or colour gradient by at least twice the
    comparator's 1e-3 of that Gaussian's own scale: one dropped row shows."""
    sc = _scene("frame-abs")
    ref = P.oracle(sc, "rgb", "none", None, False)["grads"]
    ntx = sc.views[0].ntx
    for run, (gid, (tx0, tx1, ty0, ty1), live) in sc.runs.items():
        tiles = [ty * ntx + tx for ty in range(ty0, ty1) for tx in range(tx0, tx1)]
        for k in live:
            c = _row_contrib(sc, "rgb", "none", gid, tiles[k])
            assert max(float(c[q].abs().max()) / float(ref[q][gid].abs().max()) for q in ("opa", "rgb")) >= \
                2 * P.GRAD_RTOL, (run, k)


def test_comparator_sees_faults_and_passes_fp32():
    sc = _scene("frame-abs")
    ref = P.oracle(sc, "rgb", "filt3d", None, False)
    n = sc.n
    assert P.compare(n, ref["grads"], ref["grads"]) == []
    gid, (tx0, tx1, ty0, ty1), live = sc.runs["siteA"]
    ntx = sc.views[0].ntx
    tiles = [ty * ntx + tx for ty in range(ty0, ty1) for tx in range(tx0, tx1)]
    row = {q: g[gid] for q, g in P.oracle(sc, "rgb", "filt3d", None, False, tiles=[tiles[live[1]]])["grads"].items()}
    other = {q: g[gid] for q, g in P.oracle(sc, "rgb", "filt3d", None, False, tiles=[tiles[live[0]]])["grads"].items()}
    for name, delta in (("dropped", {q: -row[q] for q in row}), ("duplicated", row),
                        ("stale", {q: other[q] - row[q] for q in row})):
        bad = {q: g.clone() for q, g in ref["grads"].items()}
        for q in bad:
            bad[q][gid] += delta[q]
        assert P.compare(n, bad, ref["grads"]) != [], name
    # a row where the oracle's is exactly zero (a visible, unbinned Gaussian)
    unb = sc.roles.index("unbinned")
    assert all(float(g[unb].abs().max()) == 0 for g in ref["grads"].values())
    bad = {q: g.clone() for q, g in ref["grads"].items()}
    bad["pos"][unb] += row["pos"]
    assert P.compare(n, bad, ref["grads"]) != []
    # the 3-D filter's backward left out
    un = P.oracle(sc, "rgb", "filt3d", None, False, unchained=True)
    assert any(f.startswith("scale") for f in P.compare(n, un["grads"], ref["grads"]))
    # fp32 evaluation of the same oracle passes
    r32 = P.oracle(sc, "rgb", "filt3d", None, False, dtype=torch.float32)
    assert P.compare(n, r32["grads"], ref["grads"], r32["images"], ref["images"], r32["cam"], ref["cam"]) == []
