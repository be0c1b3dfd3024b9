#!/usr/bin/env python
"""View-sharded data-parallel training loop on a synthetic multi-view scene (SURVEY.md §8f-1,
the multi-view training configuration): the `train_step` of the reference trainer (train.py:85-201 — zero_grad,
render one training camera, L1 loss, backward, Adam over the five parameter groups with the
reference's learning-rate factors train.py:21-25,56-64) with the one change multi-GPU needs: each
rank renders a different view and the gradients are all-reduced (one flat bucket) before the step.

  python examples/train_dp.py --gaussians 200000 --res 640x360 --iters 300
  python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_dp.py ...
  python examples/train_dp.py --surfel --lambda-normal 0.05 --lambda-dist 100    # 2D Gaussian Splatting
  python examples/train_dp.py --prune-at 100 --prune-keep 0.5     # keep the half that blends the most weight

Ground truth = renders of a "teacher" Gaussian set; the student starts from perturbed positions,
grey colours and low opacity.  Prints loss / PSNR and iterations per second.
"""
import argparse
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

import dp  # noqa: E402
import loss as L  # noqa: E402
import optim  # noqa: E402
import splatter  # noqa: E402
import synthetic as S  # noqa: E402


def build(n, w, h, n_views, dev, seed=0, student_kw=None):
    teacher = S.make_gaussians(n, w, h, seed)
    views = [S.make_view(w, h, k) for k in range(n_views)]
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    prim = (student_kw or {}).get("primitive", "gaussian")        # the teacher renders the student's primitive
    sp_t = splatter.Splatter.from_tensors(teacher, vd, device=dev, primitive=prim)
    with torch.no_grad():
        gts = [sp_t(k).clone() for k in range(n_views)]
    g = torch.Generator().manual_seed(seed + 100)          # identical on every rank: replicas start equal
    student = {k: v.clone() for k, v in teacher.items()}
    student["pos"] += torch.randn(n, 3, generator=g) * 0.01
    student["rgb"] = torch.zeros_like(teacher["rgb"])
    student["opa"] = torch.full_like(teacher["opa"], -2.0)
    student["scale"] = teacher["scale"] * (1 + 0.2 * torch.randn(n, 3, generator=g)).clamp(0.5, 1.5)
    return splatter.Splatter.from_tensors(student, vd, device=dev, **(student_kw or {})), gts


def make_optimizer(sp, lr=0.003, fused=True):
    g = sp.gaussian_3ds
    cls = optim.FlatAdam if fused else torch.optim.Adam             # FlatAdam: one kernel over the flat bucket
    return cls([                                                     # train.py:56-64
        {"params": g.opa, "lr": lr * 10}, {"params": g.rgb, "lr": lr * 10}, {"params": g.pos, "lr": lr},
        {"params": g.scale, "lr": lr}, {"params": g.quat, "lr": lr}], betas=(0.9, 0.99))


def train(sp, gts, iters, world, rank, log_every=50, lr=0.003, fused_adam=True, visible_adam=False, cap_max=None,
          filter3d_every=0, lambda_normal=0.0, lambda_dist=0.0, prune_at=None, prune_keep=1.0):
    opt = make_optimizer(sp, lr, fused_adam)
    params = list(sp.gaussian_3ds.parameters())
    surfel = sp.primitive == "surfel"
    # peer-memory exchange when available, else NCCL; surfel frames have no gradient push, so they all-reduce
    bucket = dp.make_grad_bucket(params, average=True, exchange="nccl" if surfel else "auto")
    maps = surfel and (lambda_normal > 0 or lambda_dist > 0)
    mc = None
    if cap_max is not None:                                           # MCMC densification, refining every 100 steps
        import mcmc
        mc = mcmc.MCMC(sp, opt, cap_max, refine_start=min(500, iters // 4), refine_stop=max(iters - 100, 0))
    hist = []
    torch.cuda.synchronize()
    t0 = time.time()
    for it in range(iters):
        opt.zero_grad(set_to_none=True)
        view = dp.view_for_rank(it, rank, world, len(gts))
        if maps:                                                      # 2DGS: L1 + normal consistency + distortion
            out = sp.render_surfel_maps(view)
            img = out["image"]
            v = sp.current_view
            loss = ((img - gts[view]).abs().mean()
                    + lambda_normal * L.surfel_normal_consistency(out["normal"], out["depth"], out["alpha"],
                                                                  v["focal_x"], v["focal_y"])
                    + lambda_dist * out["distortion"].mean())
        else:
            img = sp(view)
            loss = (img - gts[view]).abs().mean()                    # train.py:99
        loss.backward()
        bucket.allreduce()
        if mc is not None:                                            # after the exchange: every rank adds the same
            mc.after_backward(it)
        if visible_adam:                                              # step only the Gaussians some rank binned
            opt.step(visible=dp.all_reduce_visible(sp.visible_mask()))
        else:
            opt.step()
        if filter3d_every and it % filter3d_every == 0:                 # Mip-Splatting: over all training views
            sp.compute_filter3d()
        if it == prune_at:                                            # LightGaussian-style: by summed blend weight
            scores = sp.score_views(range(rank, len(gts), world))     # this rank's share of the training views
            if world > 1:                                             # summed over the shares: every view once
                scores.all_reduce()
            n = sp.gaussian_3ds.pos.shape[0]
            top = torch.sort(scores.weight_sum, descending=True, stable=True).indices[:max(1, int(prune_keep * n))]
            sp.prune(torch.zeros(n, dtype=torch.bool, device=top.device).index_fill_(0, top, True), opt)
            bucket.params = list(sp.gaussian_3ds.parameters())
        if mc is not None:
            n = sp.gaussian_3ds.pos.shape[0]
            mc.after_step(it, lr)
            if sp.gaussian_3ds.pos.shape[0] != n:                     # grown: the exchange follows the new Parameters
                bucket.params = list(sp.gaussian_3ds.parameters())
        if it % log_every == 0 or it == iters - 1:
            with torch.no_grad():
                mse = ((img - gts[view]) ** 2).mean()
                psnr = float(-10 * torch.log10(mse + 1e-12))
            hist.append((it, float(loss), psnr))
            if rank == 0:
                print(f"iter {it:5d}  L1 {float(loss):.5f}  PSNR {psnr:6.2f} dB  view {view}  "
                      f"n {sp.gaussian_3ds.pos.shape[0]}", flush=True)
    torch.cuda.synchronize()
    return hist, iters / (time.time() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=200_000)
    ap.add_argument("--res", default="640x360")
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--views", type=int, default=8)
    ap.add_argument("--torch-adam", action="store_true", help="use torch.optim.Adam instead of the fused flat Adam")
    ap.add_argument("--visible-adam", action="store_true",
                    help="update only the Gaussians binned this step (3DGS sparse Adam); unseen ones stay frozen")
    ap.add_argument("--mcmc", action="store_true",
                    help="MCMC densification (3DGS-MCMC, mcmc.MCMC): relocate dead Gaussians and grow to --cap-max "
                         "every 100 steps, position noise every step; with --visible-adam the opacity and scale "
                         "regularisers reach only the visible rows, like every other gradient")
    ap.add_argument("--cap-max", type=int, default=None, help="Gaussian count cap of --mcmc (default 1.5 x --gaussians)")
    ap.add_argument("--filter3d", action="store_true",
                    help="Mip-Splatting's configuration: the 2-D antialias filter and the 3-D filter (variance 0.1), "
                         "recomputed every 100 steps over all training views on every rank")
    ap.add_argument("--surfel", action="store_true",
                    help="2D Gaussian Splatting: train (and render the ground truth with) surfels")
    ap.add_argument("--lambda-normal", type=float, default=0.0, help="--surfel: weight of the normal-consistency loss")
    ap.add_argument("--lambda-dist", type=float, default=0.0, help="--surfel: weight of the depth-distortion loss")
    ap.add_argument("--prune-at", type=int, default=None,
                    help="at this step, score every training view (each rank its share, all-reduced) and keep the "
                         "--prune-keep fraction of the Gaussians with the largest summed blend weight "
                         "(Splatter.score_views / prune)")
    ap.add_argument("--prune-keep", type=float, default=0.5, help="--prune-at: fraction of the Gaussians kept")
    args = ap.parse_args()
    if args.prune_at is not None and args.surfel:
        ap.error("--prune-at scores 3-D Gaussian frames; it does not take --surfel")
    if not 0.0 < args.prune_keep <= 1.0:
        ap.error("--prune-keep must be in (0, 1]")
    if (args.lambda_normal or args.lambda_dist) and not args.surfel:
        ap.error("--lambda-normal / --lambda-dist need --surfel")
    if args.surfel and args.filter3d:
        ap.error("--surfel takes no --filter3d")
    if args.visible_adam and args.torch_adam:
        ap.error("--visible-adam is a mode of the fused flat Adam")
    if args.cap_max is not None and not args.mcmc:
        ap.error("--cap-max needs --mcmc")
    w, h = (int(x) for x in args.res.split("x"))
    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=dev)
    torch.manual_seed(2023)                                           # identical torch RNG on all ranks
    kw = dict(filter2d="antialias", filter3d=True, filter3d_variance=0.1) if args.filter3d else None
    if args.surfel:
        kw = dict(primitive="surfel")
    sp, gts = build(args.gaussians, w, h, args.views, dev, student_kw=kw)
    hist, ips = train(sp, gts, args.iters, world, rank, fused_adam=not args.torch_adam,
                      visible_adam=args.visible_adam,
                      cap_max=(args.cap_max or int(1.5 * args.gaussians)) if args.mcmc else None,
                      filter3d_every=100 if args.filter3d else 0, lambda_normal=args.lambda_normal,
                      lambda_dist=args.lambda_dist, prune_at=args.prune_at, prune_keep=args.prune_keep)
    if rank == 0:
        print(f"done: {ips:.1f} it/s ({ips * world:.1f} views/s on {world} GPU), L1 {hist[0][1]:.5f} -> {hist[-1][1]:.5f}, "
              f"PSNR {hist[0][2]:.2f} -> {hist[-1][2]:.2f} dB, {sp.gaussian_3ds.pos.shape[0]} Gaussians")
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
