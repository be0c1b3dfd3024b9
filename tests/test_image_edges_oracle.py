"""CPU checks of tests/image_edges.py: the loss and bilateral-grid fixtures reach their design (every tile-position
residue of the loss's inner band and last tile, the round-up knot pixels of every GL that has them, the slice's
launch-split counts), the torch fp32 restatements of both kernels pass the per-element comparators on every
fixture, and deliberately wrong fp32 variants fail them: the loss's inner band one pixel too wide, a halo tap lost on
tiles' last columns, sign(0) taken as +1; the slice's z cell from a plain floorf and a missing cell-boundary row."""
import numpy as np
import pytest
import torch

import bilagrid_oracle as BO
import image_edges as E
import loss_oracle as LO


# ------------------------------------------------------------------------------------------------------------- loss
def test_loss_shapes_cover_every_tile_position():
    hs = {h for h, w in E.LOSS_SHAPES}
    ws = {w for h, w in E.LOSS_SHAPES}
    for dims in (hs, ws):
        assert set(E.RESIDUES) <= {d % E.TILE for d in dims if d > E.TILE}
        assert set(range(12, 17)) <= dims
    assert (11, 2000) in E.LOSS_SHAPES and (2000, 11) in E.LOSS_SHAPES and E.UHD == (2160, 3840)


@pytest.mark.parametrize("half", [False, True], ids=["f32", "f16"])
def test_loss_contents_reach_their_design(half):
    h, w = 47, 37
    x, y = E.loss_pair(h, w, "flat", half)
    yd = y.double()
    assert x.dtype == torch.float32 and y.dtype == (torch.float16 if half else torch.float32)
    assert bool((x == 0).any()) and bool((yd == 1).any())
    for c, a in ((0.98, 1e-3), (0.999, 1e-5)):
        near = (x.double() - c).abs() <= a * 1.01
        assert int(near.all(-1).sum()) > 100
    x, y = E.loss_pair(h, w, "equal", half)
    eq = x.double() == y.double()
    assert 0.3 < float(eq.double().mean()) < 0.7
    x, y = E.loss_pair(h, w, "checker", half)
    assert set(torch.unique(x).tolist()) == {0.0, 1.0}
    x, y = E.loss_pair(h, w, "impulse", half)
    sites = E.impulse_sites(h, w)
    moved = {tuple(p) for p in torch.nonzero((x.double() != y.double()).any(-1)).tolist()}
    assert moved == set(sites)
    assert {(15, 15), (16, 16), (E.HALF, w // 3), (h - E.HALF - 1, w // 3), (h // 3, E.HALF - 1)} <= moved
    x, y = E.loss_pair(130, 200, "mixed", half)
    assert x.shape == (130, 200, 3) and bool((x.double() == y.double()).any())
    assert bool((x[:64, :64] == E.loss_pair(130, 200, "flat", half, seed=0)[0][:64, :64]).all())


def test_ssim_terms_match_the_definition_and_autograd():
    x, y = E.loss_pair(38, 47, "noise")
    xd, yd = x.double().requires_grad_(True), y.double()
    t = LO.ssim_terms(xd.detach(), yd)
    s = LO.ssim(xd, yd)
    s.backward()
    n_inner = 3 * 28 * 37
    assert abs(float(t["s"].sum()) / n_inner - float(s)) < 1e-14
    assert float((t["grad"] / n_inner - xd.grad).abs().max()) < 1e-14 * float(xd.grad.abs().max()) * 100
    for k in ("A", "B", "C"):
        assert bool((t[k + "_mag"] >= t[k].abs()).all()), k
    assert bool((t["grad_mag"] >= t["grad"].abs()).all())


def _value_excess(ref, mode, result):
    """|value - oracle| / bound of the total, and for the SSIM-weighted calls of the SSIM mean alone"""
    (total, _, ss), _ = result
    v, vb = ref.value(mode)
    r = abs(total - v) / vb if vb > 0 else float(total != v) * float("inf")
    if ss is not None and E.loss_weights(mode)[1] != 0:
        r = max(r, abs(ss - ref.ssim) / ref.ssim_bound())
    return r


def _grad_excess(ref, mode, result):
    g, gb = ref.grad(mode)
    return E.excess(result[1], g, gb)


LOSS_CASES = [(h, w, c, half) for (h, w) in E.LOSS_SHAPES for c in E.CONTENTS for half in (False, True)]


@pytest.mark.parametrize("h,w,content,half", LOSS_CASES,
                         ids=[f"{h}x{w}-{c}-{'f16' if hf else 'f32'}" for h, w, c, hf in LOSS_CASES])
def test_loss_comparator_passes_fp32_and_fails_wrong_variants(h, w, content, half):
    """The value and the gradient comparators each on their own: fp32 passes both; the inner band one pixel too wide
    fails both (the value on every call that weights SSIM); a lost halo tap and sign(0) = +1 touch the gradient only."""
    x, y = E.loss_pair(h, w, content, half)
    ref = E.LossRef(x, y)
    for mode in E.CALLS:
        args = E.loss_weights(mode)
        # the oracle's formula evaluated in fp32 through autograd, and the kernel's arithmetic restated in fp32
        xa = x.clone().requires_grad_(True)
        tot = args[0] * (xa - y.float()).abs().mean() + args[1] * LO.ssim(xa, y.float()) + args[2]
        tot.backward()
        autograd = ((float(tot.detach()), None, None), xa.grad)
        restated = E.loss_fp32(x, y, *args)
        for res in (autograd, restated):
            assert _value_excess(ref, mode, res) <= 1.0, mode
            assert _grad_excess(ref, mode, res) <= 1.0, mode
        band = E.loss_fp32(x, y, *args, band=1)
        if args[1] != 0:
            assert _value_excess(ref, mode, band) > 1.0, mode
            assert _grad_excess(ref, mode, band) > 1.0, mode
    args = E.loss_weights("w=0.1")
    halo = _grad_excess(ref, "w=0.1", E.loss_fp32(x, y, *args, drop_halo_tap=True))
    # seen wherever a tile's last column has its right halo inside the image and a gradient around it (the impulses
    # of a strip 11 rows high lie on the inner band's edges only, away from those columns)
    if w > E.TILE and (content != "impulse" or h > E.TILE):
        assert halo > 1.0
    elif w <= E.TILE:
        assert halo <= 1.0
    sign0 = _grad_excess(ref, "w=0.1", E.loss_fp32(x, y, *args, sign0=1.0))
    if content in ("equal", "checker", "impulse"):             # x == y over whole regions
        assert sign0 > 1.0
    elif not bool((x.double() == y.double()).any()):
        assert sign0 <= 1.0


# --------------------------------------------------------------------------------------------------- bilateral grid
def test_roundup_knots_are_exactly_the_listed_ones():
    assert {gl: E.roundup_knots(gl) for gl in range(2, 17) if E.roundup_knots(gl)} == E.ROUNDUP_KNOTS


@pytest.mark.parametrize("gl", sorted(E.ROUNDUP_KNOTS))
def test_roundup_pixels_sit_below_their_knot(gl):
    px = E.roundup_knot_pixels(gl, 40, seed=gl)
    z = BO.guide_f32(px)
    exact = z.astype(np.float64) * (gl - 1)
    prod = exact.astype(np.float32)
    assert np.all(prod == np.round(prod)) and np.all(exact < prod)                    # rounds up onto a knot
    assert set(np.round(prod).astype(int).tolist()) == set(E.ROUNDUP_KNOTS[gl])
    assert np.all(E.plain_floor_cell(z, gl) == E.exact_cell(z, gl) + 1)
    # the oracle's exact cell is the lower one
    z0, _, _ = BO._zcell(torch.from_numpy(z.astype(np.float64)), gl)
    assert np.all(z0.numpy() == E.exact_cell(z, gl))


@pytest.mark.parametrize("name", [n for n in E.SLICE_BUILDERS if n.startswith(("knots", "roundup"))])
def test_knot_fixtures_mix_knots_with_black_white_and_out_of_range(name):
    case = E.SLICE_BUILDERS[name]()
    gl = case.grids.shape[3]
    z = BO.guide_f32(case.image)
    assert (z == 0).any() and (z == 1).any() and (z < 0).any() and (z > 1).any()
    inside = (z > 0) & (z < 1)
    if name.startswith("knots"):
        assert np.all((z[inside] * (gl - 1)) == np.round(z[inside] * (gl - 1)))
    else:
        differ = E.plain_floor_cell(z, gl) != E.exact_cell(z, gl)
        assert differ.sum() == inside.sum() > 100


def test_slice_fixtures_reach_the_launch_splits_and_grid_edges():
    B = {n: len(E.SLICE_BUILDERS[n]().ids) for n in ("fwd-B64", "fwd-B65", "fwd-B129", "B65535")}
    assert B == {"fwd-B64": 64, "fwd-B65": 65, "fwd-B129": 129, "B65535": 65535}
    assert {(n + E.FWD_IDS_PER_LAUNCH - 1) // E.FWD_IDS_PER_LAUNCH for n in B.values()} >= {1, 2, 3}
    for name, n in (("table-960", 960), ("table-961", 961)):
        c = E.SLICE_BUILDERS[name]()
        assert len(c.ids) + len(c.views) == n and c.ids != sorted(c.ids)
    c = E.SLICE_BUILDERS["B65535"]()
    assert len(c.ids) + len(c.views) > E.TABLE_PER_LAUNCH and c.image.shape[1:3] == (1, 2)
    c = E.SLICE_BUILDERS["cells-over-pixels"]()
    assert c.grids.shape[1:4] == (256, 256, 16) and (c.grids.shape[1] - 1) * (c.grids.shape[2] - 1) > 45 * 67
    c = E.SLICE_BUILDERS["one-pixel-cells"]()
    assert c.grids.shape[1] - 1 == c.image.shape[1] and c.grids.shape[2] - 1 == c.image.shape[2]
    c = E.SLICE_BUILDERS["lattice-through-centres"]()
    gx = (np.arange(4) + 0.5) * (c.grids.shape[2] - 1) / 4
    assert np.all(gx == np.round(gx))
    c = E.SLICE_BUILDERS["one-cell-tall"]()
    assert c.grids.shape[1:3] == (2, 2) and c.image.shape[1] < E.MAX_SLICES / 2 and c.image.shape[1] > c.image.shape[2]
    for n in E.SLICE_BUILDERS:
        c = E.SLICE_BUILDERS[n]()
        assert len(c.views) < c.grids.shape[0], n          # some view's grad row must be left alone


@pytest.mark.parametrize("name", list(E.SLICE_BUILDERS))
def test_slice_comparator_passes_fp32_and_fails_wrong_variants(name):
    case = E.SLICE_BUILDERS[name]()
    ref = E.SliceRef(case)
    assert max(E.slice_excess(ref, case, *E.slice_fp32(case))) <= 1.0
    floor = max(E.slice_excess(ref, case, *E.slice_fp32(case, plain_floor=True)))
    assert (floor > 1.0) == name.startswith("roundup"), floor
    gh = case.grids.shape[1]
    rows = len(set(E._fma_free_cells(case.image.shape[1], gh)[0].tolist()))
    row = max(E.slice_excess(ref, case, *E.slice_fp32(case, skip_cell_row=True)))
    assert (row > 1.0) == (rows > 1), row
