"""CPU fp64 restatement of MCMC densification (3DGS-MCMC; gsplat's MCMCStrategy) as gs_mcmc_relocate / gs_mcmc_add /
gs_mcmc_noise define it in include/gs_b200.h.  The sampler's uniforms and the noise's z are inputs, so the device
results can be compared draw by draw.  Arrays are numpy; parameters come in as float32 and go out as float32, the
arithmetic in between is fp64."""
import math

import numpy as np

MAX_RATIO = 51


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, dtype=np.float64)))


def activate(raw, act):
    raw = np.asarray(raw, dtype=np.float64)
    return np.abs(raw) + 1e-4 if act == "abs" else np.exp(raw)


def ratio(o, r):
    """(o', den, coefficient o / den) for a source of opacity o with ratio r: the double sum exactly as written.  r = 1
    is the identity, exactly (1 - (1 - o) rounds)."""
    if r == 1:
        return o, o, 1.0
    o_new = 1.0 - (1.0 - o) ** (1.0 / r)
    den = 0.0
    for a in range(1, r + 1):
        for b in range(a):
            den += math.comb(a - 1, b) * (-1) ** b * o_new ** (b + 1) / math.sqrt(b + 1)
    return o_new, den, (o / den if den > 0 else 1.0)


def weights(o):
    """round(o 2^32) as uint64 (round half to even), the sampler's fixed-point weights."""
    return np.rint(np.asarray(o, dtype=np.float64) * 2.0 ** 32).astype(np.uint64)


def sample(w, u, tol=64):
    """src_j = min{i : C_i > t_j}, t_j = min(floor(u_j C_{n-1}), C_{n-1} - 1) (the product in fp64), with C the integer
    inclusive prefix sum of the uint64 weights w.  Returns (src, near): near[j] is True when t_j lies within `tol`
    units of the prefix sums around it.  The sums are exact, so the device's C equals this one unless its fp64
    sigmoid put some o_i 2^32 on the other side of a half (each such weight moves the later C_i by one unit); `tol`
    bounds how many of those a comparison allows before a draw's index may legitimately differ."""
    w = np.asarray(w, dtype=np.uint64)
    C = np.cumsum(w, dtype=np.uint64)
    total = C[-1]
    t = np.floor(np.asarray(u, dtype=np.float32).astype(np.float64) * np.float64(total)).astype(np.uint64)
    t = np.minimum(t, total - np.uint64(1))
    src = np.searchsorted(C, t, side="right")
    hi = C[src].astype(np.int64)
    lo = np.where(src > 0, C[np.maximum(src - 1, 0)], 0).astype(np.int64)
    ti = t.astype(np.int64)
    near = (hi - ti <= tol) | (ti - lo < tol)
    return src, near


def new_opa_scale(opa, scale, i, r, act, min_opacity):
    """float32 (logit, raw scale [3]) that source i with ratio r and every copy of it get."""
    o = float(sigmoid(opa[i]))
    o_new, _, coef = ratio(o, r)
    o_new = min(max(o_new, min_opacity), 1.0 - 2.0 ** -23)
    logit = np.float32(math.log(o_new / (1.0 - o_new)))
    raw = np.asarray(scale[i], dtype=np.float64)
    s_new = coef * activate(raw, act)
    if act == "abs":
        sign = np.where(np.asarray(scale[i]) < 0, -1.0, 1.0)
        raw_new = sign * np.maximum(s_new - 1e-4, 0.0)
    else:
        raw_new = np.log(s_new)
    return logit, raw_new.astype(np.float32)


def _apply(params, src, dst, act, min_opacity, out):
    counts = np.bincount(src, minlength=len(params["opa"]))
    for j, (i, t) in enumerate(zip(src, dst)):
        r = min(1 + int(counts[i]), MAX_RATIO)
        logit, raw = new_opa_scale(params["opa"], params["scale"], i, r, act, min_opacity)
        for k, a in params.items():
            if a is not None:
                out[k][t] = a[i]
        out["opa"][t] = logit
        out["scale"][t] = raw
        out["opa"][i] = logit
        out["scale"][i] = raw
    return counts


def relocate(params, act, min_opacity, u):
    """params: dict of float32 arrays pos [n,3], rgb [n,d], opa [n], quat [n,4], scale [n,3], feat [n,f] or None.
    Returns (new params, touched bool [n], n_relocated, near-boundary flags of the draws)."""
    min_opacity = float(np.float32(min_opacity))
    o = sigmoid(params["opa"])
    dead = o <= min_opacity
    out = {k: (None if a is None else a.copy()) for k, a in params.items()}
    touched = np.zeros(len(o), dtype=bool)
    w = np.where(dead, np.uint64(0), weights(o))
    k = int(dead.sum())
    if k == 0 or int(w.sum()) == 0:
        return out, touched, 0, np.zeros(0, dtype=bool)
    dst = np.nonzero(dead)[0]
    src, near = sample(w, np.asarray(u)[:k])
    _apply(params, src, dst, act, min_opacity, out)
    touched[src] = True
    touched[dst] = True
    return out, touched, k, near


def add(params, act, min_opacity, u):
    """len(u) Gaussians appended, drawn over all with weight o.  Returns (new params of n + len(u) rows, src, near)."""
    min_opacity = float(np.float32(min_opacity))
    n, n_new = len(params["opa"]), len(u)
    out = {k: (None if a is None else np.concatenate([a, np.zeros((n_new,) + a.shape[1:], a.dtype)]))
           for k, a in params.items()}
    w = weights(sigmoid(params["opa"]))
    if int(w.sum()) == 0:                          # nothing to draw from: plain copies of row 0
        for k, a in params.items():
            if a is not None:
                out[k][n:] = a[0]
        return out, np.zeros(n_new, dtype=np.int64), np.zeros(n_new, dtype=bool)
    src, near = sample(w, u)
    _apply(params, src, n + np.arange(n_new), act, min_opacity, out)
    return out, src, near


def gate(opa):
    return 1.0 / (1.0 + np.exp(-100.0 * ((1.0 - sigmoid(opa)) - 0.995)))


def quat_to_rot(q):
    q = np.asarray(q, dtype=np.float64)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * z * w, 2 * x * z + 2 * y * w,
                     2 * x * y + 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * x * w,
                     2 * x * z - 2 * y * w, 2 * y * z + 2 * x * w, 1 - 2 * x * x - 2 * y * y], -1).reshape(
                         q.shape[:-1] + (3, 3))


def noise_delta(quat, scale, opa, act, scaler, z):
    """The displacement scaler g(o) R diag(s^2) R^T z, fp64 [n, 3]."""
    R = quat_to_rot(quat)
    s2 = activate(scale, act) ** 2
    a = s2 * np.einsum("nji,nj->ni", R, np.asarray(z, dtype=np.float64))   # diag(s^2) R^T z
    return scaler * gate(opa)[:, None] * np.einsum("nij,nj->ni", R, a)


def regularizer_grads(opa, scale, act, opacity_reg, scale_reg):
    """d/d(opa, raw scale) of opacity_reg mean(sigmoid(opa)) + scale_reg mean(s)."""
    n = len(opa)
    o = sigmoid(opa)
    ds = np.exp(np.asarray(scale, np.float64)) if act == "exp" else np.sign(np.asarray(scale, np.float64))
    return opacity_reg / n * o * (1 - o), scale_reg / (3 * n) * ds
