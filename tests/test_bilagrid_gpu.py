"""The bilateral-grid slice kernels (csrc/bilagrid.cu) against the fp64 oracle, their determinism, the autograd chain
through a render and the loss, checkpoints, and a short appearance-jittered training run."""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

import bilagrid_oracle as BO

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _image(b, h, w, seed, dev):
    """values in [-0.1, 1.1], with rows of pure black and pure white pixels"""
    g = torch.Generator().manual_seed(seed)
    x = -0.1 + 1.2 * torch.rand(b, h, w, 3, generator=g)
    x[:, ::7] = 0.0
    x[:, 3::11] = 1.0
    return x.to(dev)


def _grids(v, shape, seed, dev):
    return BO.random_grids(v, *shape, seed=seed).float().to(dev)


def _rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max() / (b.double().abs().max() + 1e-30))


def _go(shape, seed, dev):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(dev)


CASES = [((1080, 1920), 1, [0]), ((45, 67), 1, [1]), ((8, 5), 1, [1]), ((45, 67), 4, [2, 0, 2, 1])]


@pytest.mark.parametrize("shape", [(16, 16, 8), (8, 4, 4), (2, 2, 2), (4, 6, 16), (5, 3, 11)])
@pytest.mark.parametrize("hw,b,ids", CASES, ids=["1920x1080", "67x45", "5x8", "67x45-B4-repeat"])
def test_kernel_matches_oracle(gs, cuda, shape, hw, b, ids):
    gaussian, _ = gs
    if hw[0] == 1080 and shape not in ((16, 16, 8), (8, 4, 4), (2, 2, 2)):
        pytest.skip("the 1080p case runs the three main grid shapes")
    img = _image(b, *hw, seed=sum(hw) + b, dev=cuda)
    grids = _grids(3, shape, seed=b, dev=cuda)
    out = gaussian.bilagrid_slice(img, grids, ids)
    ref = BO.slice_forward(img.double().cpu(), grids.double().cpu(), ids)
    assert float((out.double().cpu() - ref).abs().max()) <= 1e-5
    go = _go(img.shape, 3, cuda)
    gi, gg = gaussian.bilagrid_slice_backward(img, grids, ids, go, True, True)
    ri, rg = BO.slice_backward(img.double().cpu(), grids.double().cpu(), ids, go.double().cpu())
    assert _rel(gi, ri) <= 1e-4
    assert _rel(gg, rg) <= 1e-4
    untouched = [v for v in range(3) if v not in ids]
    for v in untouched:
        assert torch.count_nonzero(gg[v]) == 0


def test_single_image_and_batch_agree(gs, cuda):
    gaussian, _ = gs
    img = _image(2, 40, 50, seed=5, dev=cuda)
    grids = _grids(2, (8, 8, 4), seed=6, dev=cuda)
    go = _go(img.shape, 7, cuda)
    out = gaussian.bilagrid_slice(img, grids, [1, 0])
    assert torch.equal(out[1], gaussian.bilagrid_slice(img[1].contiguous(), grids, [0]))
    gi, _ = gaussian.bilagrid_slice_backward(img, grids, [1, 0], go, True, False)
    gi1, _ = gaussian.bilagrid_slice_backward(img[1].contiguous(), grids, [0], go[1].contiguous(), True, False)
    assert torch.equal(gi[1], gi1)


def test_identity_grids_return_the_input(gs, cuda):
    import bilagrid
    gaussian, _ = gs
    img = torch.rand(2, 1080, 1920, 3, generator=torch.Generator().manual_seed(8)).to(cuda)
    for shape in ((16, 16, 8), (3, 7, 13)):
        grids = bilagrid.identity_grids(3, shape, cuda)
        out = gaussian.bilagrid_slice(img, grids, [2, 0])
        assert float((out - img).abs().max()) <= 1e-6


def test_backward_is_bit_deterministic(gs, cuda):
    gaussian, _ = gs
    img = _image(2, 1080, 1920, seed=9, dev=cuda)
    grids = _grids(2, (16, 16, 8), seed=10, dev=cuda)
    go = _go(img.shape, 11, cuda)
    a = gaussian.bilagrid_slice_backward(img, grids, [1, 1], go, True, True)
    b = gaussian.bilagrid_slice_backward(img, grids, [1, 1], go, True, True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("shape", [(16, 16, 8), (4, 4, 3), (6, 5, 16)])
def test_partial_calls_match_the_full_call(gs, cuda, shape):
    gaussian, _ = gs
    img = _image(3, 100, 130, seed=12, dev=cuda)
    grids = _grids(2, shape, seed=13, dev=cuda)
    go = _go(img.shape, 14, cuda)
    gi, gg = gaussian.bilagrid_slice_backward(img, grids, [0, 1, 0], go, True, True)
    gi_only, none_g = gaussian.bilagrid_slice_backward(img, grids, [0, 1, 0], go, True, False)
    none_i, gg_only = gaussian.bilagrid_slice_backward(img, grids, [0, 1, 0], go, False, True)
    assert torch.equal(gi, gi_only) and torch.equal(gg, gg_only)
    assert none_g is None and none_i is None


def test_refusals_through_the_binding(gs, cuda):
    gaussian, _ = gs
    img = _image(1, 16, 16, seed=15, dev=cuda)
    with pytest.raises(RuntimeError, match="outside"):
        gaussian.bilagrid_slice(img, _grids(2, (4, 4, 4), 0, cuda), [2])
    with pytest.raises(RuntimeError, match="grid dimensions"):
        gaussian.bilagrid_slice(img, _grids(1, (4, 4, 17), 0, cuda), [0])
    with pytest.raises(RuntimeError, match="one view id per image"):
        gaussian.bilagrid_slice(img, _grids(2, (4, 4, 4), 0, cuda), [0, 1])


def _restated_slice(image, grids, view):
    """torch restatement on the device: grid_sample + affine, z from the kernel's fp32 expression"""
    img = image[None]
    h, w = image.shape[:2]
    lum = BO.LUM[0] * img[..., 0] + BO.LUM[1] * img[..., 1] + BO.LUM[2] * img[..., 2]
    z = torch.from_numpy(BO.guide_f32(img)).to(image.device) + (lum - lum.detach())
    xs = ((torch.arange(w, device=image.device, dtype=torch.float32) + 0.5) / w).expand(1, h, w)
    ys = ((torch.arange(h, device=image.device, dtype=torch.float32) + 0.5) / h)[:, None].expand(1, h, w)
    coords = torch.stack([xs, ys, z], dim=-1)[:, None] * 2 - 1
    A = torch.nn.functional.grid_sample(grids.permute(0, 4, 3, 1, 2)[view:view + 1], coords, mode="bilinear",
                                        padding_mode="border", align_corners=True)[:, :, 0].permute(0, 2, 3, 1)
    return BO.apply_affine(A, img)[0]


def _scene(cuda, n=20000, w=256, h=256, n_views=4):
    import splatter
    import synthetic as S
    g = S.make_gaussians(n, w, h, seed=3)
    views = [S.make_view(w, h, k) for k in range(n_views)]
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    return splatter.Splatter.from_tensors(g, vd, device=cuda)


def test_chain_through_render_and_loss_matches_restatement(gs, cuda):
    import bilagrid
    import loss as L
    sp = _scene(cuda)
    gt = torch.rand(256, 256, 3, generator=torch.Generator().manual_seed(16)).to(cuda)
    bg = bilagrid.BilateralGrids(4, (8, 8, 4), device=cuda)
    with torch.no_grad():
        bg.grids.add_(0.1 * torch.randn(bg.grids.shape, generator=torch.Generator().manual_seed(17)).to(cuda))
    grads = []
    for fn in (lambda im: bg(im, 2), lambda im: _restated_slice(im, bg.grids, 2)):
        for p in list(sp.gaussian_3ds.parameters()) + [bg.grids]:
            p.grad = None
        L.l1_ssim_loss(fn(sp(2)), gt)[0].backward()
        grads.append({k: getattr(sp.gaussian_3ds, k).grad.clone() for k in ("pos", "rgb", "opa", "quat", "scale")}
                     | {"grids": bg.grids.grad.clone()})
    for k in grads[0]:
        assert _rel(grads[0][k], grads[1][k]) <= 1e-3, k


def test_checkpoint_restores_grids_and_moments(gs, cuda, tmp_path):
    import bilagrid
    import checkpoint
    sp = _scene(cuda, n=2000, w=64, h=64, n_views=2)
    bg = bilagrid.BilateralGrids(2, (4, 4, 4), device=cuda)
    opt = torch.optim.Adam(bg.parameters(), lr=2e-3, eps=1e-15)
    for v in (0, 1, 0):
        opt.zero_grad()
        (bg(sp(v).detach(), v) ** 2).mean().backward()
        opt.step()
    path = str(tmp_path / "ckpt.pth")
    checkpoint.save_checkpoint(sp, path, bilagrid=bg, bilagrid_optimizer=opt)
    bg2 = bilagrid.BilateralGrids(2, (4, 4, 4), device=cuda)
    opt2 = torch.optim.Adam(bg2.parameters(), lr=2e-3, eps=1e-15)
    checkpoint.load_checkpoint(path, sp, bilagrid=bg2, bilagrid_optimizer=opt2)
    assert torch.equal(bg.grids, bg2.grids)
    s1, s2 = opt.state[bg.grids], opt2.state[bg2.grids]
    for k in ("exp_avg", "exp_avg_sq", "step"):
        assert torch.equal(s1[k].cpu(), s2[k].cpu()), k
    # a file without grids leaves the module as it is
    path0 = str(tmp_path / "plain.pth")
    checkpoint.save_checkpoint(sp, path0)
    bg3 = bilagrid.BilateralGrids(2, (4, 4, 4), device=cuda)
    checkpoint.load_checkpoint(path0, sp, bilagrid=bg3)
    assert torch.equal(bg3.grids, bilagrid.identity_grids(2, (4, 4, 4), cuda))


def test_grids_absorb_appearance_jitter_in_training(gs, cuda):
    """8 views with jittered ground truth: training with grids fits the jittered views better (lower training L1) than
    training without.  The colour-corrected PSNR of the raw renders against the clean views is printed and checked to
    be finite, not compared: at this length the grids did not raise it (29.80 against 30.33 dB on an H100, DESIGN.md
    section 5)."""
    import bilagrid
    import synthetic as S
    spec = importlib.util.spec_from_file_location("train_dp", os.path.join(ROOT, "examples", "train_dp.py"))
    td = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(td)
    res = {}
    for use in (False, True):
        torch.manual_seed(2023)
        sp, clean = td.build(20000, 256, 256, 8, cuda)
        gts = S.appearance_jitter(clean, 0.3, seed=1)
        bg = bilagrid.BilateralGrids(8, device=cuda) if use else None
        hist, _ = td.train(sp, gts, 400, 1, 0, log_every=1, bilagrid_module=bg)
        l1 = float(np.mean([h[1] for h in hist[-40:]]))
        res[use] = (l1, td.cc_psnr(sp, clean))
    print(f"train L1 / colour-corrected PSNR vs clean: without grids {res[False][0]:.5f} / {res[False][1]:.2f} dB, "
          f"with grids {res[True][0]:.5f} / {res[True][1]:.2f} dB")
    assert res[True][0] < res[False][0]
    assert math.isfinite(res[True][1]) and math.isfinite(res[False][1])
