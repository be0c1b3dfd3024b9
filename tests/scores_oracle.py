"""fp64 restatement of the blend-weight scores (gs_frame_scores, `Splatter.score_views`), on top of gs_oracle's `draw`
arithmetic: for Gaussian i and pixel p of the cropped image, w = alpha T with T the exclusive transmittance while
T >= 1e-4 (else 0), alpha = opa exp(power) as `draw` forms them.  weight_sum[i] = sum_p w, weight_max[i] = max_p w.

`weights` scores already sorted instances; `scores` runs a front end first: gs_oracle's (through filter_oracle, which
adds the 2-D filter), or lens_oracle's culling with a lens."""
import torch

import filter_oracle as F
import gs_oracle as O
import lens_oracle as LO


def crop_box(cam):
    """(left, top, width, height) of the rendered image inside the padded one (splatter.py:267-272)."""
    return (cam.Wp - cam.width) // 2, (cam.Hp - cam.height) // 2, cam.width, cam.height


def weights(pos, opa, cov, accum, gauss_idx, n, Hp, Wp, fx, fy, crop=None):
    """(weight_sum[n], weight_max[n], npix[n]) of sorted instances (pos[M, 2+], opa[M], cov[M, 2, 2], tile ranges accum
    [T+1], gauss_idx[M] their Gaussians) in fp64.  crop: (left, top, width, height), None = the whole padded image.
    npix[i]: the image pixels of the tiles Gaussian i was binned into (the scale of its weight_sum's rounding)."""
    dt = torch.float64
    pos, opa, cov = pos.detach().to(dt), opa.detach().to(dt), cov.detach().to(dt).reshape(-1, 4)
    accum = accum.to(torch.int64)
    gauss_idx = gauss_idx.to(torch.int64)
    left, top, cw, ch = crop if crop is not None else (0, 0, Wp, Hp)
    ntx = Wp // 16
    ix = torch.arange(16)
    ws = torch.zeros(n, dtype=dt)
    wm = torch.zeros(n, dtype=dt)
    npix = torch.zeros(n, dtype=dt)
    for t in range(accum.numel() - 1):
        s, e = int(accum[t]), int(accum[t + 1])
        if e <= s:
            continue
        ty, tx = divmod(t, ntx)
        gx, gy = tx * 16 + ix, ty * 16 + ix
        px = (gx.to(dt) + 0.5 - (Wp // 2)) / fx
        py = (gy.to(dt) + 0.5 - (Hp // 2)) / fy
        PX = px.reshape(1, 16).expand(16, 16).reshape(-1, 1)
        PY = py.reshape(16, 1).expand(16, 16).reshape(-1, 1)
        inx = (gx >= left) & (gx < left + cw)
        iny = (gy >= top) & (gy < top + ch)
        inb = (iny.reshape(16, 1) & inx.reshape(1, 16)).reshape(-1, 1).to(dt)
        a, b, c, d = cov[s:e].unbind(-1)
        X = PX - pos[s:e, 0].reshape(1, -1)
        Y = PY - pos[s:e, 1].reshape(1, -1)
        det = a * d - b * c
        alpha = torch.exp(-(d * X * X - (b + c) * X * Y + a * Y * Y) / (2 * det + 1e-14)) * opa[s:e].reshape(1, -1)
        Tinc = torch.cumprod(1 - alpha, dim=1)
        Texc = torch.cat([torch.ones(256, 1, dtype=dt), Tinc[:, :-1]], dim=1)
        w = alpha * Texc * (Texc >= 0.0001).to(dt) * inb
        gi = gauss_idx[s:e]
        ws.index_add_(0, gi, w.sum(0))
        wm.scatter_reduce_(0, gi, w.amax(0), reduce="amax")
        npix.index_add_(0, gi, inb.sum().expand(e - s))
    return ws, wm, npix


def scores(g, cam, mode="none", variance=0.3, lens=None, depth_key=None, thresh=0.05):
    """weights() of the frame of parameters g (dict pos, rgb, opa, quat, scale; abs scale activation) through camera
    cam: with the 2-D filter `mode` / `variance`, or through `lens` (dict(model, cx, cy, k); no 2-D filter)."""
    dt = torch.float64
    p = {q: t.detach().to(dt) for q, t in g.items()}
    rgb3 = torch.zeros(p["pos"].shape[0], 3, dtype=dt)          # the colour does not enter the weights
    n = p["pos"].shape[0]
    if lens is None:
        pos, _, opa, cov, accum, _, _, gidx = F._front(p["pos"], rgb3, p["opa"], p["quat"], p["scale"], cam, mode,
                                                       variance, thresh, "abs", False, depth_key)
    else:
        assert mode == "none"
        rot, tran = cam.rot.to(dt), cam.tran.to(dt)
        nq, ns, opa_a, _ = O.preactivate(p["quat"], p["scale"], p["opa"], rgb3, "abs", False)
        ox, oy = LO.offsets(lens, cam.width, cam.height, cam.fx, cam.fy)
        rp, rc, mask = LO.global_culling_lens(p["pos"], nq, ns, rot, tran, cam.near, cam.half_w, cam.half_h, lens,
                                              ox, oy)
        idx = torch.nonzero(mask.bool()).squeeze(-1)
        p_c, c_c = rp[idx], rc[idx]
        rects = O.tile_rects(p_c[:, :2], c_c, thresh, cam.tile_lx, cam.tile_ly, cam.ntx, cam.nty, cam.leftmost,
                             cam.topmost)
        gi, accum = O.bin_and_sort(p_c, c_c, rects, cam.ntx, cam.nty, None if depth_key is None else depth_key[idx])
        pos, opa, cov, gidx = p_c[gi], opa_a[idx][gi], c_c[gi], idx[gi]
    return weights(pos, opa, cov, accum, gidx, n, cam.Hp, cam.Wp, cam.fx, cam.fy, crop_box(cam))
