"""loss.surfel_normal_consistency: the value on a tilted plane, and its gradient with respect to the normal, depth
and alpha maps against central differences."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

import loss  # noqa: E402

H, W, F = 12, 14, 30.0


def _plane():
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    qx = (xs + 0.5 - W / 2) / F
    z = 2.0 / (1 - 0.3 * qx)                  # the plane z - 0.3 x_c = 2 (x_c = qx z)
    n = torch.tensor([0.3, 0.0, -1.0], dtype=torch.float64)
    return z, n / n.norm()


def test_value_on_a_plane():
    z, n = _plane()
    alpha = torch.full((H, W), 0.8, dtype=torch.float64)
    normal = alpha[..., None] * n                 # sum w n of an opaque-enough surface
    val = loss.surfel_normal_consistency(normal, alpha * z, alpha, F, F)
    assert abs(float(val) - (1 - 0.8 * 0.8)) < 1e-9
    val1 = loss.surfel_normal_consistency(torch.ones(H, W, 1, dtype=torch.float64) * n, z, torch.ones(H, W,
                                          dtype=torch.float64), F, F)
    assert abs(float(val1)) < 1e-9


def test_gradients_match_central_differences():
    z, n = _plane()
    g = torch.Generator().manual_seed(0)
    alpha = 0.5 + 0.4 * torch.rand(H, W, generator=g, dtype=torch.float64)
    depth = alpha * z * (1 + 0.05 * torch.rand(H, W, generator=g, dtype=torch.float64))
    normal = alpha[..., None] * n + 0.1 * torch.randn(H, W, 3, generator=g, dtype=torch.float64)
    ins = [normal.clone().requires_grad_(True), depth.clone().requires_grad_(True)]
    loss.surfel_normal_consistency(ins[0], ins[1], alpha, F, F).backward()
    assert float(ins[1].grad.abs().max()) > 0          # the depth side is supervised too
    eps = 1e-6
    for k, t in enumerate((normal, depth)):
        for j in range(0, t.numel(), 37):
            tp, tm = t.clone(), t.clone()
            tp.view(-1)[j] += eps
            tm.view(-1)[j] -= eps
            a = [tp if k == 0 else normal, tp if k == 1 else depth]
            b = [tm if k == 0 else normal, tm if k == 1 else depth]
            fd = float(loss.surfel_normal_consistency(a[0], a[1], alpha, F, F)
                       - loss.surfel_normal_consistency(b[0], b[1], alpha, F, F)) / (2 * eps)
            assert abs(fd - float(ins[k].grad.view(-1)[j])) < 1e-6, (k, j)
