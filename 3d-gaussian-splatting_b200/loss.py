"""Training loss on the device (SURVEY.md §8 f-3): reference train.py:99-107

    l1_loss   = (rendered_img - ground_truth).abs().mean()
    ssim_loss = 1 - StructuralSimilarityIndexMeasure(data_range=1.0)(img NCHW, gt NCHW)
    loss      = (1 - ssim_weight) * l1_loss + ssim_weight * ssim_loss

as ONE autograd node over two CUDA kernels (csrc/loss.cu, C ABI `gs_loss_l1_ssim`): the forward
also produces d loss / d image, in the [H, W, 3] layout the fused blend backward consumes, so
`loss.backward()` only scales it.  `ssim` / `psnr` are the two metrics train.py evaluates
(train.py:72-73,114,265-269) for callers that keep the reference's separate L1 / SSIM terms
(the `shims/torchmetrics` package routes them here).
"""
from __future__ import annotations

import torch

import gaussian


class _L1SSIM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, target, w_l1, w_ssim, bias):
        img = image.detach()
        if img.dtype != torch.float32 or not img.is_contiguous():
            img = img.float().contiguous()
        tgt = target.detach()
        if tgt.dtype not in (torch.float32, torch.float16):
            tgt = tgt.float()
        tgt = tgt.contiguous()
        want = image.requires_grad
        out3, grad = gaussian.loss_l1_ssim(img, tgt, float(w_l1), float(w_ssim), float(bias), want)
        ctx.save_for_backward(grad if want else img.new_empty(0))
        ctx.want = want
        total, l1, ssim = out3[0], out3[1], out3[2]
        ctx.mark_non_differentiable(l1, ssim)
        return total, l1, ssim

    @staticmethod
    def backward(ctx, g_total, _g_l1, _g_ssim):
        (grad,) = ctx.saved_tensors
        return (grad * g_total if ctx.want else None), None, None, None, None


def l1_ssim_loss(image, target, ssim_weight=0.1):
    """train.py:99-107 -> (loss, l1_loss, ssim_loss); image / target [H, W, 3]."""
    w = float(ssim_weight)
    total, l1, ssim = _L1SSIM.apply(image, target, 1.0 - w, -w, w)
    return total, l1, 1.0 - ssim


def ssim(image, target):
    """Differentiable mean SSIM of two [H, W, 3] images (torchmetrics defaults, data_range = 1)."""
    return _L1SSIM.apply(image, target, 0.0, 1.0, 0.0)[0]


def l1(image, target):
    return _L1SSIM.apply(image, target, 1.0, 0.0, 0.0)[0]


def psnr(image, target, data_range=None):
    """torchmetrics PeakSignalNoiseRatio() semantics (train.py:73,114): data_range=None takes the
    target's value range."""
    t = target.to(image.dtype)
    mse = torch.mean((image - t) ** 2)
    dr = (t.max() - t.min()) if data_range is None else torch.as_tensor(float(data_range), device=image.device)
    return 10.0 * torch.log10(dr * dr / mse)


def surfel_normal_consistency(normal, depth, alpha, fx, fy, eps=1e-8):
    """2DGS's normal-consistency term on the maps of a surfel frame (renderer.render_frame_surfel): the mean over the
    interior pixels of 1 - alpha n . n_d, where n = normal [H,W,3] (sum w n, camera frame) and n_d is the unit normal of
    the surface back-projected from the expected depth depth / alpha through the pixel rays
    ((x + 0.5 - W/2) / fx, (y + 0.5 - H/2) / fy, 1), from central differences, turned to face the camera.  As in 2DGS,
    the gradient reaches both sides: the normal map, and the depth and alpha maps through n_d; the alpha weight is a
    constant."""
    h, w = depth.shape
    d = depth / alpha.clamp_min(eps)
    xs = (torch.arange(w, dtype=d.dtype, device=d.device) + 0.5 - w / 2) / fx
    ys = (torch.arange(h, dtype=d.dtype, device=d.device) + 0.5 - h / 2) / fy
    P = torch.stack([xs[None, :].expand(h, w) * d, ys[:, None].expand(h, w) * d, d], dim=-1)
    dx = P[1:-1, 2:] - P[1:-1, :-2]
    dy = P[2:, 1:-1] - P[:-2, 1:-1]
    nd = torch.linalg.cross(dy, dx, dim=-1)
    nd = nd / nd.norm(dim=-1, keepdim=True).clamp_min(eps)
    a = alpha[1:-1, 1:-1].detach()
    return (1.0 - a * (normal[1:-1, 1:-1] * nd).sum(-1)).mean()
