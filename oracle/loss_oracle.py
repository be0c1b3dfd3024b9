"""CPU oracle of the training loss (SURVEY.md §8 f-3).  TEST INFRASTRUCTURE ONLY.

reference train.py:99-107 computes  (1-w) * mean|img-gt| + w * (1 - SSIM)  with
`torchmetrics.StructuralSimilarityIndexMeasure(data_range=1.0)` (train.py:72).  torchmetrics is a
third-party dependency that is absent from /root/reference and from this image (requirements.txt
lists it unpinned), so its published algorithm is restated here from
torchmetrics/functional/image/ssim.py `_ssim_update` (v1.x; defaults gaussian_kernel=True,
kernel_size=11, sigma=1.5, k1=0.01, k2=0.03):
  * 1-D window exp(-(d/sigma)^2/2), d = -5..5, normalised; 2-D = outer product; per-channel (grouped) conv;
  * inputs reflect-padded by 5, `conv2d` of the five stacked maps (x, y, x^2, y^2, xy);
  * ssim map = ((2 mu_x mu_y + c1)(2 s_xy + c2)) / ((mu_x^2 + mu_y^2 + c1)(s_xx + s_yy + c2));
  * the same 5-pixel border is cropped from the map before the mean (so the padding never contributes);
  * mean over pixels and channels (per image, then over the batch of 1).
PARITY UNPINNED against torchmetrics itself (it cannot be installed here); the formula above is
the published one and the tests pin the CUDA kernels to this restatement in fp64 (+ finite
differences of it through autograd).
"""
import torch
import torch.nn.functional as F


def gaussian_window(kernel_size=11, sigma=1.5, dtype=torch.float64, device=None):
    dist = torch.arange((1 - kernel_size) / 2, (1 + kernel_size) / 2, 1, dtype=dtype, device=device)
    g = torch.exp(-((dist / sigma) ** 2) / 2)
    return g / g.sum()


def ssim(pred_hwc, target_hwc, data_range=1.0, k1=0.01, k2=0.03):
    """Mean SSIM of two [H, W, 3] images, torchmetrics semantics (NCHW inside)."""
    dt = pred_hwc.dtype
    x = pred_hwc.permute(2, 0, 1).unsqueeze(0)
    y = target_hwc.to(dt).permute(2, 0, 1).unsqueeze(0)
    c1, c2 = (k1 * data_range) ** 2, (k2 * data_range) ** 2
    w1 = gaussian_window(dtype=dt, device=x.device)
    ch = x.shape[1]
    kernel = (w1.unsqueeze(1) @ w1.unsqueeze(0)).expand(ch, 1, 11, 11).contiguous()
    pad = 5
    xp = F.pad(x, (pad, pad, pad, pad), mode="reflect")
    yp = F.pad(y, (pad, pad, pad, pad), mode="reflect")
    stack = torch.cat((xp, yp, xp * xp, yp * yp, xp * yp))
    out = F.conv2d(stack, kernel, groups=ch)
    mu_x, mu_y, exx, eyy, exy = out.split(1)
    sxx, syy, sxy = exx - mu_x ** 2, eyy - mu_y ** 2, exy - mu_x * mu_y
    full = ((2 * mu_x * mu_y + c1) * (2 * sxy + c2)) / ((mu_x ** 2 + mu_y ** 2 + c1) * (sxx + syy + c2))
    inner = full[..., pad:-pad, pad:-pad]
    return inner.reshape(inner.shape[0], -1).mean(-1).mean()


def train_loss(img, gt, ssim_weight=0.1):
    """train.py:99-107 -> (loss, l1_loss, ssim_loss)."""
    l1 = (img - gt.to(img.dtype)).abs().mean()
    s = 1.0 - ssim(img, gt)
    return (1 - ssim_weight) * l1 + ssim_weight * s, l1, s


def _win_valid(m, w1):
    """the 11x11 window over [N, 1, H, W] maps, at the window centres inside the image: [N, 1, H - 10, W - 10]"""
    return F.conv2d(F.conv2d(m, w1.view(1, 1, 1, -1)), w1.view(1, 1, -1, 1))


def _win_transpose(m, w1):
    """adjoint of _win_valid: spreads [N, 1, H - 10, W - 10] window-centre values back over the [N, 1, H, W] pixels"""
    return _win_valid(F.pad(m, (10, 10, 10, 10)), w1)


def ssim_terms(pred_hwc, target_hwc, c1=1e-4, c2=9e-4):
    """Per window (channel, inner centre; [3, H - 10, W - 10]) the SSIM value `s` of the definition above and its
    partial derivatives A = ds/dmu_x, B = ds/dE[x^2], C = ds/dE[xy] (the other two held), together with the
    first-order error scales of an fp32 evaluation (an fp32 result differs by a small multiple of eps times them):
      * `F` = 1 + (E[x^2] + E[y^2]) / d2: s_xx = E[x^2] - mu_x^2 and s_yy cancel to an absolute error of a few ulp of
        E[x^2] + E[y^2], which d2 = s_xx + s_yy + c2 turns into a relative one;
      * s_xy = E[xy] - mu_x mu_y cancels likewise, to an absolute error of a few ulp of |E[xy]| + |mu_x mu_y|;
      * `s_mag`, `A_mag`, `B_mag`, `C_mag`: |s| F plus n2's cancellation, and the same propagated through the terms
        of A, B and C.
    Also the image gradient of sum(s) over the windows, `grad` [H, W, 3], and its term magnitude `grad_mag`."""
    dt = pred_hwc.dtype
    x = pred_hwc.permute(2, 0, 1).unsqueeze(1)
    y = target_hwc.to(dt).permute(2, 0, 1).unsqueeze(1)
    w1 = gaussian_window(dtype=dt, device=x.device)
    mx, my, exx, eyy, exy = (_win_valid(m, w1) for m in (x, y, x * x, y * y, x * y))
    sxx, syy, sxy = exx - mx * mx, eyy - my * my, exy - mx * my
    n1, n2 = 2 * mx * my + c1, 2 * sxy + c2
    d1, d2 = mx * mx + my * my + c1, sxx + syy + c2
    dd = d1 * d2
    s = n1 * n2 / dd
    A = 2 * my * (n2 - n1) / dd - 2 * mx * s * (d2 - d1) / dd
    B = -s / d2
    C = 2 * n1 / dd
    Fc = 1 + (exx + eyy) / d2
    xy_mag = 2 * exy.abs() + 2 * (mx * my).abs()            # absolute error scale of n2, beyond its own rounding
    s_mag = s.abs() * Fc + n1.abs() * xy_mag / dd
    A_mag = 2 * my.abs() * ((n2.abs() + n1.abs()) * Fc + xy_mag) / dd + 4 * mx.abs() * s_mag * (1 / d1 + 1 / d2.abs())
    B_mag = 2 * s_mag / d2.abs()
    C_mag = 2 * n1.abs() * Fc / dd
    tA, tB, tC = (_win_transpose(m, w1) for m in (A, B, C))
    mA, mB, mC = (_win_transpose(m, w1) for m in (A_mag, B_mag, C_mag))
    grad = tA + 2 * x * tB + y * tC
    grad_mag = mA + 2 * x.abs() * mB + y.abs() * mC
    hwc = lambda m: m[:, 0].permute(1, 2, 0)                                            # noqa: E731
    return dict(s=s[:, 0], A=A[:, 0], B=B[:, 0], C=C[:, 0], F=Fc[:, 0], s_mag=s_mag[:, 0],
                A_mag=A_mag[:, 0], B_mag=B_mag[:, 0], C_mag=C_mag[:, 0], grad=hwc(grad), grad_mag=hwc(grad_mag))
