"""CPU checks of the screen-space densification statistics: the oracle of tests/densify_stats_oracle.py against
identities, a finite difference and a closed form; DensifyStats.all_reduce under gloo; and the argument checks of the
C entry points, which need no GPU."""
import ctypes
import math
import os
import socket
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import densify_stats_oracle as DS
import filter_oracle as F
import gs_oracle as O
from helpers import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "3d-gaussian-splatting_b200")


def _loss(seed):
    def f(out):
        gen = torch.Generator().manual_seed(seed)
        L = 0.0
        for k, t in out.items():
            L = L + (t * (torch.rand(t.shape, generator=gen, dtype=t.dtype) * 2 - 1)).sum()
        return L
    return f


def _small():
    g, v, cam = scene(300, 48, 32, k=1, opa_range=(0.05, 0.9))
    return {q: t.double() for q, t in g.items()}, cam


def test_pixel_contributions_sum_to_grad2d_vector():
    g, cam = _small()
    r = DS.frame_stats(*(g[q] for q in ("pos", "rgb", "opa", "quat", "scale")), cam, _loss(1))
    vis = r["count"] > 0
    assert int(vis.sum()) > 50
    scale = float(r["vec"].abs().max())
    assert float((r["pix_sum"] - r["vec"]).abs().max()) < 1e-10 * scale
    r2 = DS.frame_stats(*(g[q] for q in ("pos", "rgb", "opa", "quat", "scale")), cam, _loss(1), maps=True)
    assert float((r2["pix_sum"] - r2["vec"]).abs().max()) < 1e-10 * float(r2["vec"].abs().max())


def test_absgrad_bounds_grad2d_with_equality_for_one_pixel():
    g, cam = _small()
    r = DS.frame_stats(*(g[q] for q in ("pos", "rgb", "opa", "quat", "scale")), cam, _loss(2))
    assert bool((r["absgrad"] >= r["grad2d"] * (1 - 1e-12)).all())
    assert float((r["absgrad"] - r["grad2d"]).max()) > 0           # cancellation happens somewhere
    # only one pixel carries an upstream gradient: nothing can cancel
    py, px = 13, 21
    w = torch.tensor([0.3, -0.7, 0.5], dtype=torch.float64)
    r1 = DS.frame_stats(*(g[q] for q in ("pos", "rgb", "opa", "quat", "scale")), cam,
                        lambda out: (out["padded"][py, px] * w).sum())
    assert float(r1["grad2d"].max()) > 0
    assert torch.allclose(r1["absgrad"], r1["grad2d"], rtol=1e-12, atol=0)


def test_ndc_scale_matches_a_one_pixel_shift():
    """grad2d's x term is dL/d(NDC x): a shift of the mean by one pixel moves NDC x by 2 / W."""
    g, cam = _small()
    params = [g[q] for q in ("pos", "rgb", "opa", "quat", "scale")]
    loss = _loss(3)
    r = DS.frame_stats(*params, cam, loss)
    fr = DS._front(*params, cam, "none", 0.3, 0.05, "abs", False, None)
    i = int(torch.argmax(r["vec"][:, 0].abs() * (r["count"] > 0)))
    k = int((fr["idx"] == i).nonzero())
    sx, _ = DS.ndc_scale(cam)

    def L_at(dpix):
        m2 = fr["m2"].detach().clone()
        m2[k, 0] += dpix / cam.fx
        pos_i = torch.cat([m2[fr["gi"]], fr["p"][:, 2:].detach()], 1)
        img = O.draw(pos_i, fr["rgb"], fr["opa"], fr["cov"], fr["accum"], cam.Hp, cam.Wp, cam.fx, cam.fy)
        return float(loss(dict(padded=img)))

    eps = 1e-3
    dL_dpix = (L_at(eps) - L_at(-eps)) / (2 * eps)
    dL_dndc = dL_dpix * cam.width / 2
    assert abs(dL_dndc - float(r["vec"][i, 0]) * sx) < 1e-5 * abs(dL_dndc) + 1e-12


def test_tile_restricted_oracle_matches_the_frame_oracle():
    """tile_stats fed the frame's own binning gives frame_stats' statistics on the Gaussians of the chosen tiles."""
    g, cam = _small()
    params = [g[q] for q in ("pos", "rgb", "opa", "quat", "scale")]
    fr = DS._front(*params, cam, "none", 0.3, 0.05, "abs", False, None)
    acc = fr["accum"].long()
    tiles = [t for t in range(cam.ntx * cam.nty) if acc[t + 1] > acc[t]][::2]
    ids = [fr["idx"][fr["gi"][int(acc[t]):int(acc[t + 1])]] for t in tiles]
    mask = torch.zeros(cam.Hp, cam.Wp, 1, dtype=torch.float64)
    for t in tiles:
        ty, tx = divmod(t, cam.ntx)
        mask[ty * 16:(ty + 1) * 16, tx * 16:(tx + 1) * 16] = 1
    G = (torch.rand(cam.Hp, cam.Wp, 3, generator=torch.Generator().manual_seed(5), dtype=torch.float64) - 0.5) * mask

    def loss(out):
        return (out["padded"] * G).sum()

    full = DS.frame_stats(*params, cam, loss)
    U, part = DS.tile_stats(*params, cam, ids, tiles, loss)
    for k in ("grad2d", "absgrad", "radius"):
        assert torch.allclose(part[k], full[k][U], rtol=1e-10, atol=1e-14), k
    assert float(full["grad2d"].max()) > 0
    assert bool((part["count"] == 1).all())


def test_radius_closed_form_axis_aligned():
    """A Gaussian on the optical axis with axis-aligned scales: lambda_max = max(s_x fx / z, s_y fy / z)^2."""
    cam = O.Camera(64, 48, 60.0, 50.0, torch.eye(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64))
    z, sxy = 5.0, (0.2, 0.35)
    pos = torch.tensor([[0.0, 0.0, z]], dtype=torch.float64)
    rgb = torch.zeros(1, 3, dtype=torch.float64)
    opa = torch.tensor([2.0], dtype=torch.float64)
    quat = torch.tensor([[1.0, 0.0, 0.0, 0.0]], dtype=torch.float64)
    scale = torch.tensor([[sxy[0], sxy[1], 0.1]], dtype=torch.float64)
    r = DS.frame_stats(pos, rgb, opa, quat, scale, cam, _loss(4), absgrad=False)
    want = 3 * max((sxy[0] + 1e-4) * cam.fx / z, (sxy[1] + 1e-4) * cam.fy / z)
    assert int(r["count"][0]) == 1
    assert abs(float(r["radius"][0]) - want) < 1e-9 * want
    # with the dilation filter the covariance grows by s / f^2 on the diagonal (s px^2 in pixel units)
    rf = DS.frame_stats(pos, rgb, opa, quat, scale, cam, _loss(4), mode="dilate", absgrad=False)
    ex, ey = F.filter_eps(cam, 0.3)
    wf = 3 * math.sqrt(max((((sxy[0] + 1e-4) / z) ** 2 + ex) * cam.fx ** 2,
                           (((sxy[1] + 1e-4) / z) ** 2 + ey) * cam.fy ** 2))
    assert abs(float(rf["radius"][0]) - wf) < 1e-9 * wf


def test_scored_plan_oracle_counts():
    g, cam = _small()
    n = g["pos"].shape[0]
    gen = torch.Generator().manual_seed(7)
    accum = torch.rand(n, generator=gen, dtype=torch.float64) * 1e-3
    count = torch.randint(0, 4, (n,), generator=gen)
    radius = torch.rand(n, generator=gen, dtype=torch.float64) * 30
    hit = accum.float() / count.clamp(min=1).float() >= 2e-4
    norm = g["scale"].norm(dim=-1)
    tau = float(norm.median())
    out, info = DS.adaptive_control_stats(g["pos"], g["rgb"], g["opa"], g["quat"], g["scale"], accum, count, tau, 10.0,
                                          grad_thresh=2e-4, max_radius=radius, max_screen_px=20.0, use_split=False,
                                          z=torch.zeros(2, 0, 3, dtype=torch.float64))
    assert info["split"] == 0 and info["cloned"] > 0 and info["deleted"] > 0
    assert out[0].shape[0] == n - info["deleted"] + info["cloned"]
    kept = ~(radius.float() > 20.0) & (g["opa"] > DS.D.inverse_sigmoid(0.02)) & (norm < 10.0)
    assert info["cloned"] == int((kept & hit & (norm <= tau)).sum())
    # clones are exact copies of their source rows
    nk = int(kept.sum())
    src = kept & hit & (norm <= tau)
    assert torch.equal(out[0][nk:], g["pos"][src])


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, PKG)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import splatter
    st = splatter.DensifyStats(5, absgrad=True, device="cpu")     # no context to register with
    st.grad2d += rank + 1
    st.absgrad += 2 * (rank + 1)
    st.count += rank + 1
    st.max_radius.copy_(torch.tensor([1.0, 7.0, 3.0, 0.0, 2.0]) * (1 if rank == 0 else -1) + 4)
    st.all_reduce()
    ok = (bool((st.grad2d == 3).all()) and bool((st.absgrad == 6).all()) and bool((st.count == 3).all())
          and st.count.dtype == torch.int32
          and torch.equal(st.max_radius, torch.tensor([5.0, 11.0, 7.0, 4.0, 6.0])))
    st.reset(3)
    ok = ok and st.n == 3 and float(st.grad2d.abs().sum()) == 0 and int(st.count.sum()) == 0
    out[rank] = 1 if ok else 0
    dist.destroy_process_group()


def test_densify_stats_all_reduce_gloo():
    ctx = mp.get_context("spawn")
    out = ctx.Array("i", [0, 0])
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
    assert all(p.exitcode == 0 for p in procs)
    assert list(out) == [1, 1]


def test_c_entry_points_reject_bad_arguments_without_a_gpu():
    lib = ctypes.CDLL(os.path.join(PKG, "libgs_b200.so"))
    lib.gs_last_error.restype = ctypes.c_char_p
    P, I, F = ctypes.c_void_p, ctypes.c_int, ctypes.c_float

    class Stats(ctypes.Structure):
        _fields_ = [("n", I), ("grad2d", P), ("absgrad", P), ("count", P), ("max_radius", P)]

    lib.gs_ctx_set_densify_stats.argtypes = [P, ctypes.POINTER(Stats)]
    s = Stats(4, 16, None, 32, 48)
    assert lib.gs_ctx_set_densify_stats(None, ctypes.byref(s)) == -1
    assert b"null ctx" in lib.gs_last_error()
    assert lib.gs_ctx_set_densify_stats(None, None) == -1
    lib.gs_densify_workspace_bytes.restype = ctypes.c_size_t
    lib.gs_densify_plan_stats.argtypes = [P, P, P, P, P, F, I, I, F, F, F, F, I, I, P, P, P, ctypes.c_size_t, P]
    args = lambda n, ws, opa=16, mr=None, px=20.0: (opa, 16, 16, 16, mr, px, n, 0, -3.9, 10.0, 2e-4, 0.05, 1, 1, 16,
                                                      16, 16, ws, None)
    assert lib.gs_densify_plan_stats(*args(-1, 1 << 20)) == -1
    assert lib.gs_densify_plan_stats(*args(10, 1 << 20, opa=None)) == -1
    assert b"bad arguments" in lib.gs_last_error()
    assert lib.gs_densify_plan_stats(*args(10, 0)) == -1
    assert b"workspace too small" in lib.gs_last_error()
    assert lib.gs_densify_plan_stats(*args(10, 1 << 20, mr=16, px=float("nan"))) == -1
    assert b"NaN" in lib.gs_last_error()
    assert lib.gs_densify_plan_stats(*args(0, lib.gs_densify_workspace_bytes(0))) == 0
