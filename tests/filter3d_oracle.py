"""CPU oracle of Mip-Splatting's 3-D smoothing filter on the fused frame path (gs_ctx_set_filter3d,
gs_filter3d_compute, `Splatter(..., filter3d=True)`).

Test infrastructure only, with no blend code of its own.  Two parts:

- `sampling_filter`: the per-Gaussian maximal sampling rate over a set of views, in fp64 from the float32 inputs.
  View c sees Gaussian i when, with p_c = R pos_i + t, u = fx x / z + W / 2 and w = fy y / z + H / 2:
  z > near, -m W <= u <= (1 + m) W and -m H <= w <= (1 + m) H.  nu_i = max over those views of fx / z and
  f_i = sqrt(v) / nu_i; an unseen Gaussian gets nu = min of the seen nu (the largest filter); none seen: f = 0.
- `filtered` / `applied`: the filtered activations s' = sqrt(s^2 + f^2) and sigma' = sigma prod s / s' (rows with
  f == 0 keep s and sigma by selection), applied to gs_oracle.preactivate's outputs.  Inside `applied(f3d)` every
  frame of filter_oracle (render / render_maps, any mode of the 2-D filter) and gs_oracle renders with the 3-D filter;
  with f == 0 everywhere it is their computation bit for bit.
"""
from __future__ import annotations

import contextlib
import math

import numpy as np
import torch

import gs_oracle as O


def sampling_filter(pos, cams, margin=0.15, variance=0.2):
    """(f [n] float64, seen [n] bool) for pos [n, 3] and cams: dicts with width, height, focal_x, focal_y, rot [3, 3],
    tran [3], near (the values the device receives: float32 where gs_camera holds float32)."""
    p = np.asarray(pos, dtype=np.float32).astype(np.float64)
    n = p.shape[0]
    m = float(np.float32(margin))
    nu = np.zeros(n)
    for c in cams:
        R = np.asarray(c["rot"], dtype=np.float32).astype(np.float64).reshape(3, 3)
        t = np.asarray(c["tran"], dtype=np.float32).astype(np.float64).reshape(3)
        W, H = float(c["width"]), float(c["height"])
        fx, fy = float(np.float32(c["focal_x"])), float(np.float32(c["focal_y"]))
        near = float(np.float32(c["near"]))
        pc = p @ R.T + t
        z = pc[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = fx * pc[:, 0] / z + W / 2
            w = fy * pc[:, 1] / z + H / 2
            seen = (z > near) & (u >= -m * W) & (u <= (1 + m) * W) & (w >= -m * H) & (w <= (1 + m) * H)
            nu = np.maximum(nu, np.where(seen, fx / z, 0.0))
    seen = nu > 0
    if not seen.any():
        return np.zeros(n), seen
    nu = np.where(seen, nu, nu[seen].min())
    return math.sqrt(float(np.float32(variance))) / nu, seen


def boundary_ties(pos, cams, margin=0.15, tol=2e-6):
    """[n] bool: Gaussians within a relative `tol` of a view's near plane or margin edge in any view, where a float32
    test (the device's) and the fp64 one may disagree; test scenes drop them."""
    p = np.asarray(pos, dtype=np.float32).astype(np.float64)
    m = float(np.float32(margin))
    tie = np.zeros(p.shape[0], dtype=bool)
    for c in cams:
        R = np.asarray(c["rot"], dtype=np.float32).astype(np.float64).reshape(3, 3)
        t = np.asarray(c["tran"], dtype=np.float32).astype(np.float64).reshape(3)
        W, H = float(c["width"]), float(c["height"])
        fx, fy = float(np.float32(c["focal_x"])), float(np.float32(c["focal_y"]))
        near = float(np.float32(c["near"]))
        pc = p @ R.T + t
        z = pc[:, 2]
        tie |= np.abs(z - near) <= tol * (np.abs(z) + near)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = fx * pc[:, 0] / z + W / 2
            w = fy * pc[:, 1] / z + H / 2
        front = z > near
        for val, lo, hi, span in ((u, -m * W, (1 + m) * W, W), (w, -m * H, (1 + m) * H, H)):
            tol_px = tol * (np.abs(val) + span)
            tie |= front & ((np.abs(val - lo) <= tol_px) | (np.abs(val - hi) <= tol_px))
    return tie


def filtered(scale_a, opa_a, f3d):
    """(s' [n, 3], sigma' [n]) from the activated scale and opacity; f3d [n] is a constant."""
    f = f3d.to(scale_a.dtype).detach()
    on = f != 0
    sf = torch.sqrt(scale_a * scale_a + (f * f).unsqueeze(1))
    ratio = torch.prod(scale_a / sf, dim=1)
    return torch.where(on.unsqueeze(1), sf, scale_a), torch.where(on, opa_a * ratio, opa_a)


@contextlib.contextmanager
def applied(f3d):
    """Within the block, gs_oracle.preactivate (and so gs_oracle / filter_oracle / aux_oracle frames) returns the
    3-D filtered scale and opacity."""
    orig = O.preactivate

    def pre(quat, scale, opa, rgb, scale_activation="abs", use_sh_coeff=False):
        nq, ns, o, c = orig(quat, scale, opa, rgb, scale_activation, use_sh_coeff)
        ns, o = filtered(ns, o, f3d)
        return nq, ns, o, c

    O.preactivate = pre
    try:
        yield
    finally:
        O.preactivate = orig


def scale_grad(g_sf, g_l2o, s, f):
    """The device's chain (gs_filter3d_backward) in float64: dL/ds from dL/ds', dL/dl2o (l2o = log2 sigma'), s, f."""
    s, f = np.asarray(s, dtype=np.float64), np.asarray(f, dtype=np.float64)[..., None]
    sf = np.sqrt(s * s + f * f)
    comp = np.where((g_l2o[..., None] != 0) & (s > 0), g_l2o[..., None] * f * f / (math.log(2) * s * (s * s + f * f)),
                    0.0)
    return np.where(f != 0, g_sf * s / sf + comp, g_sf)
