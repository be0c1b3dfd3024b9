"""The fp64 MCMC oracle (tests/mcmc_oracle.py) checked against itself and against independent evaluations: the ratio
formula's identities, its cancelling sum against 50-digit decimal arithmetic, the sampler on hand-made weights, the
noise with an identity covariance, and the regulariser gradients against autograd.  CPU only."""
import decimal
import math

import numpy as np
import pytest
import torch

import mcmc_oracle as MO

O_GRID = [1e-4, 0.005, 0.01, 0.05, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99, 0.999]


def test_ratio_one_is_the_identity():
    for o in O_GRID:
        o_new, den, coef = MO.ratio(o, 1)
        assert o_new == o and den == o and coef == 1.0


@pytest.mark.parametrize("r", range(1, 52))
def test_r_copies_compose_to_the_original_opacity(r):
    for o in O_GRID:
        o_new, _, _ = MO.ratio(o, r)
        assert abs(1 - (1 - o_new) ** r - o) <= 1e-12, (o, r)


def _den_decimal(o_new, r):
    decimal.getcontext().prec = 50
    x = decimal.Decimal(o_new)
    den = decimal.Decimal(0)
    for a in range(1, r + 1):
        for b in range(a):
            den += math.comb(a - 1, b) * (-1) ** b * x ** (b + 1) / decimal.Decimal(b + 1).sqrt()
    return den


@pytest.mark.parametrize("r", [2, 5, 11, 26, 51])
def test_den_against_fifty_digit_decimal(r):
    worst = 0.0
    for o in O_GRID:
        o_new, den, _ = MO.ratio(o, r)
        exact = _den_decimal(o_new, r)
        rel = abs(decimal.Decimal(den) - exact) / abs(exact)
        worst = max(worst, float(rel))
    assert worst < 1e-10, worst


def test_sampler_on_hand_made_weights():
    w = np.array([0, 0, 1, 0, 0, 3, 0, 4, 0], dtype=np.uint64)          # C = 0 0 1 1 1 4 4 8 8
    u = np.array([0.0, 0.124999, 0.125, 0.3, 0.49999, 0.5, 0.75, 0.999999], dtype=np.float32)
    src, near = MO.sample(w, u, tol=0)
    # t = floor(u * 8): 0 -> the first C > 0 is index 2; 1 (exactly C_2) -> index 5; 4 (exactly C_5) -> index 7
    assert src.tolist() == [2, 2, 5, 5, 5, 7, 7, 7]
    assert not near.any()
    assert all(w[s] > 0 for s in src)
    _, near = MO.sample(w, u, tol=1)                                     # t on (or one below) a prefix sum
    assert near.tolist() == [True, True, True, False, True, True, False, True]


def test_sampler_weights_are_fixed_point_and_exact():
    o = np.array([0.5, 2.0 ** -33, 2.0 ** -33 * 1.0000001, 1.0 - 2.0 ** -40, 0.25 + 2.0 ** -34])
    assert MO.weights(o).tolist() == [2 ** 31, 0, 1, 2 ** 32, 2 ** 30]   # round half to even
    w = MO.weights(np.full(2 ** 20, 0.999))
    C = np.cumsum(w, dtype=np.uint64)
    assert int(C[-1]) == int(w[0]) * 2 ** 20                              # no rounding in the sum
    src, _ = MO.sample(w, np.array([np.float32(1) - np.float32(2 ** -24)], dtype=np.float32))
    assert src.tolist() == [2 ** 20 - 1]                                  # t stays below the total


def test_relocation_moves_every_dead_gaussian_and_conserves_nothing_else():
    rng = np.random.default_rng(0)
    n = 50
    p = dict(pos=rng.normal(size=(n, 3)).astype(np.float32), rgb=rng.normal(size=(n, 3)).astype(np.float32),
             opa=rng.normal(0, 3, size=n).astype(np.float32), quat=rng.normal(size=(n, 4)).astype(np.float32),
             scale=rng.normal(-3, 1, size=(n, 3)).astype(np.float32), feat=None)
    p["opa"][:10] = -8.0                                                  # dead: sigmoid(-8) < 0.005
    out, touched, k, _ = MO.relocate(p, "exp", 0.005, rng.random(n).astype(np.float32))
    assert k == int((MO.sigmoid(p["opa"]) <= np.float32(0.005)).sum()) >= 10
    assert touched[:10].all()
    assert (MO.sigmoid(out["opa"]) >= np.float32(0.005) * (1 - 1e-6)).all()
    for key in ("pos", "rgb", "quat"):
        assert np.array_equal(out[key][~touched], p[key][~touched])


def test_noise_with_identity_rotation_and_unit_scale_is_scaler_gate_z():
    rng = np.random.default_rng(1)
    n = 100
    quat = np.tile([1.0, 0.0, 0.0, 0.0], (n, 1))
    scale = np.zeros((n, 3))                                              # exp(0) = 1
    opa = rng.normal(0, 4, size=n)
    z = rng.normal(size=(n, 3))
    d = MO.noise_delta(quat, scale, opa, "exp", 0.37, z)
    assert np.allclose(d, 0.37 * MO.gate(opa)[:, None] * z, rtol=1e-14, atol=0)
    assert MO.gate(np.array([-20.0]))[0] == pytest.approx(1 / (1 + math.exp(-0.5)), rel=1e-6)


@pytest.mark.parametrize("act", ["abs", "exp"])
def test_regulariser_gradients_match_autograd(act):
    gen = torch.Generator().manual_seed(2)
    opa = torch.randn(1000, generator=gen, dtype=torch.float64, requires_grad=True)
    scale = torch.randn(1000, 3, generator=gen, dtype=torch.float64, requires_grad=True)
    s = scale.abs() + 1e-4 if act == "abs" else scale.exp()
    loss = 0.01 * torch.sigmoid(opa).mean() + 0.02 * s.mean()
    loss.backward()
    go, gs = MO.regularizer_grads(opa.detach().numpy(), scale.detach().numpy(), act, 0.01, 0.02)
    assert np.allclose(go, opa.grad.numpy(), rtol=1e-12, atol=0)
    assert np.allclose(gs, scale.grad.numpy(), rtol=1e-12, atol=0)
