"""Per-view bilateral grids for appearance correction (Wang et al., "Bilateral Guided Radiance Field Processing",
SIGGRAPH Asia 2024).

Photos of one capture differ in exposure, white balance and tone curve from shot to shot.  A small learned grid per
training image, a lattice over (x, y, luminance) whose nodes hold 3x4 affine colour transforms, absorbs those
differences: during training the render is sliced through its view's grid before the loss, so the Gaussians are left
to model the scene.  Test views render without a grid.

The slice is one autograd node over two CUDA kernels (csrc/bilagrid.cu, C ABI `gs_bilagrid_slice_fwd` / `_bwd`; the
definition and the grid layout [V, GH, GW, GL, 12] are in include/gs_b200.h).  Its grid gradient is bit-deterministic.

    bg = BilateralGrids(n_views, device=dev)
    bg_opt = torch.optim.Adam(bg.parameters(), lr=2e-3, eps=1e-15)
    img = bg(sp(view), view)                           # [H, W, 3], or [B, H, W, 3] with B view ids
    loss = l1_ssim_loss(img, gt)[0] + 10.0 * bg.tv_loss([view])
"""
from __future__ import annotations

from typing import Iterable, Sequence, Union

import torch


def _ids(view_ids) -> list:
    if isinstance(view_ids, int):
        return [view_ids]
    if torch.is_tensor(view_ids):
        return [int(v) for v in view_ids.reshape(-1).tolist()]
    return [int(v) for v in view_ids]


class _Slice(torch.autograd.Function):
    @staticmethod
    def forward(ctx, image, grids, ids):
        import gaussian
        img = image.detach().float().contiguous()
        out = gaussian.bilagrid_slice(img, grids.detach(), ids)
        ctx.save_for_backward(img, grids.detach())
        ctx.ids = ids
        return out

    @staticmethod
    def backward(ctx, grad_out):
        import gaussian
        img, grids = ctx.saved_tensors
        gi, gg = gaussian.bilagrid_slice_backward(img, grids, ctx.ids, grad_out.float().contiguous(),
                                                  ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return (gi if ctx.needs_input_grad[0] else None), (gg if ctx.needs_input_grad[1] else None), None


def slice_image(image, grids, view_ids):
    """image [H, W, 3] with one view id, or [B, H, W, 3] with B ids (repeats allowed); grids [V, GH, GW, GL, 12].
    Differentiable in both."""
    ids = _ids(view_ids)
    n = 1 if image.dim() == 3 else image.shape[0]
    if len(ids) != n:
        raise ValueError(f"bilagrid.slice_image: {n} image(s) but {len(ids)} view id(s)")
    return _Slice.apply(image, grids, ids)


def identity_grids(n_views, shape=(16, 16, 8), device=None):
    gh, gw, gl = shape
    eye = torch.tensor([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=torch.float32, device=device)
    return eye.expand(n_views, gh, gw, gl, 12).contiguous()


class BilateralGrids(torch.nn.Module):
    """One bilateral grid per training view: `grids` [n_views, GH, GW, GL, 12], initialised to the identity."""

    def __init__(self, n_views: int, shape=(16, 16, 8), device=None):
        super().__init__()
        self.shape = tuple(int(s) for s in shape)
        self.grids = torch.nn.Parameter(identity_grids(int(n_views), self.shape, device))

    @property
    def n_views(self) -> int:
        return self.grids.shape[0]

    def forward(self, image, view_ids: Union[int, Sequence[int], torch.Tensor]):
        return slice_image(image, self.grids, view_ids)

    def tv_loss(self, view_ids: Iterable[int]):
        """Total variation of the given views' grids: the mean squared difference between neighbouring nodes along y,
        x and the luminance axis, summed over the three axes."""
        rows = [self.grids[v:v + 1] for v in sorted(set(_ids(view_ids)))]       # basic slices: no index upload
        return tv_loss(rows[0] if len(rows) == 1 else torch.cat(rows))

    @torch.no_grad()
    def all_reduce_grad(self, view_ids: Iterable[int], group=None):
        """SUM the gradient rows of `view_ids` across ranks.  Pass every view rendered in this step on ANY rank (the
        same list on every rank).  Each view's row is written by the rank that rendered it, so the sum is that rank's
        gradient; an average would shrink it by the world size.  The other rows are left as they are."""
        rows = torch.tensor(sorted(set(_ids(view_ids))), device=self.grids.device)
        if self.grids.grad is None:
            self.grids.grad = torch.zeros_like(self.grids)
        g = self.grids.grad.index_select(0, rows)
        torch.distributed.all_reduce(g, op=torch.distributed.ReduceOp.SUM, group=group)
        self.grids.grad.index_copy_(0, rows, g)


def tv_loss(grids):
    """grids [n, GH, GW, GL, 12] -> mean squared neighbour difference along GH + along GW + along GL."""
    dy = grids[:, 1:] - grids[:, :-1]
    dx = grids[:, :, 1:] - grids[:, :, :-1]
    dz = grids[:, :, :, 1:] - grids[:, :, :, :-1]
    return dy.square().mean() + dx.square().mean() + dz.square().mean()


@torch.no_grad()
def color_correct(image, target):
    """The least-squares 3x4 affine colour fit of `image` to `target` (both [..., 3]), applied to `image`.  The
    evaluation metric of appearance-corrected models: PSNR(color_correct(render, gt), gt) fits out one global colour
    transform per image before comparing.  Solved in float64; returned in the image's dtype."""
    x = image.reshape(-1, 3).double()
    t = target.reshape(-1, 3).double()
    xa = torch.cat([x, torch.ones_like(x[:, :1])], dim=1)
    m = torch.linalg.solve(xa.T @ xa, xa.T @ t)
    return (xa @ m).reshape(image.shape).to(image.dtype)
