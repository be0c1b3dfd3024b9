"""MCMC densification at C3 size (2.4 M Gaussians): the position noise, relocation and growth kernels, and a training
step with and without MCMC's per-step work.

In one process, on the GPU (no device: it fails, there is no fallback):
  * a 1 GiB device-to-device copy timed with CUDA events: the HBM bandwidth this card reaches (read + written bytes);
  * the noise kernel (gs_mcmc_noise, Philox z and caller-given z) against its torch restatement (randn, quaternion
    to matrix, batched products), on bench.py's C3 scene; algorithmic bytes 56 N (44 read, 12 written) for the
    Philox kernel, 68 N with a given z;
  * relocation with 5 % of the Gaussians dead (gs_mcmc_relocate with FlatAdam-layout moments): each timed call first
    restores the opacities (a 9.6 MB copy, timed alone and reported), so every call relocates the same 5 %;
  * growth by 5 % (gs_mcmc_add: the copy of the n rows into the new arrays and the draws);
  * a training step (frame forward + backward, FlatAdam) with and without MCMC's every-step work (regulariser
    gradients + noise), RGB colour at view 0, alternated by round.
Variants are alternated inside every round; a round times --launches calls per variant between two CUDA events; the
figure is the median of --rounds rounds.  The card's name and power limit are read (query only) and printed with the
numbers.  Human-readable lines go to stderr, one JSON line to stdout.

  python examples/bench_mcmc.py [--launches 20] [--rounds 5] [--e2e-steps 20]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))
sys.path.insert(0, os.path.join(ROOT, "examples"))

import gaussian  # noqa: E402
import optim  # noqa: E402
import splatter  # noqa: E402
import synthetic as S  # noqa: E402
from bench_optim import BETAS, N, W, H, card, copy_gbs, layout, log, median, time_variants, views_dict  # noqa: E402

SCALER = 0.01


def scene(dev):
    g = S.make_gaussians(N, W, H, 0, sh_dim=3, opa_range=(0.05, 0.9))
    return {k: t.to(dev).contiguous() for k, t in g.items()}


def torch_noise(p, scaler, gen):
    """The noise in torch, as a trainer without the kernel would write it."""
    o = torch.sigmoid(p["opa"])
    gate = torch.sigmoid(-100.0 * ((1 - o) - 0.995))
    R = splatter.quat_to_rotmat(p["quat"] / p["quat"].norm(dim=-1, keepdim=True))
    s = p["scale"].abs() + 1e-4
    cov = (R * (s * s).unsqueeze(-2)) @ R.transpose(-1, -2)
    z = torch.randn(p["pos"].shape, device=p["pos"].device, generator=gen)
    p["pos"].add_(scaler * gate.unsqueeze(-1) * (cov @ z.unsqueeze(-1)).squeeze(-1))


def bench_noise(dev, launches, rounds, gbs):
    p = scene(dev)
    z = torch.randn(N, 3, device=dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    seeds = iter(range(1 << 30))
    variants = {
        "kernel_philox": lambda: gaussian.mcmc_noise(p["pos"], p["quat"], p["scale"], p["opa"], 0, SCALER, next(seeds)),
        "kernel_given_z": lambda: gaussian.mcmc_noise(p["pos"], p["quat"], p["scale"], p["opa"], 0, SCALER, 0, z),
        "torch": lambda: torch_noise(p, SCALER, gen),
    }
    times = time_variants(variants, launches, rounds)
    rows = []
    for k, ts in times.items():
        ms = median(ts)
        row = {"variant": k, "ms": round(ms, 4), "ms_rounds": [round(t, 4) for t in ts]}
        if k.startswith("kernel"):
            nbytes = (56 if k == "kernel_philox" else 68) * N
            rate = nbytes / (ms * 1e-3) / 1e9
            row.update(MB=round(nbytes / 1e6, 1), GBps=round(rate, 1), share_of_copy=round(rate / gbs, 3))
        rows.append(row)
        log(f"noise {k:<15} {ms:8.4f} ms" + (f"  {row['GBps']:7.0f} GB/s  {row['share_of_copy']:6.1%} of copy"
                                               if "GBps" in row else ""))
    del p, z
    torch.cuda.empty_cache()
    return rows


def bench_refine(dev, launches, rounds):
    p = scene(dev)
    gen = torch.Generator().manual_seed(1)
    dead = torch.rand(N, generator=gen) < 0.05
    p["opa"][dead.to(dev)] = -8.0
    opa0 = p["opa"].clone()
    starts, widths, total = layout(N, 3)
    m, v = torch.randn(total, device=dev), torch.rand(total, device=dev)
    u = torch.rand(N, device=dev)
    u_add = torch.rand(int(1.05 * N) - N, device=dev)

    def relocate():
        p["opa"].copy_(opa0)
        gaussian.mcmc_relocate(p["pos"], p["rgb"], p["opa"], p["quat"], p["scale"], None, 0, 0.005, u, exp_avg=m,
                               exp_avg_sq=v, seg_starts=starts, seg_widths=widths)

    def grow():
        gaussian.mcmc_add(p["pos"], p["rgb"], opa0, p["quat"], p["scale"], None, 0, 0.005, u_add)

    times = time_variants({"restore_opa_only": lambda: p["opa"].copy_(opa0), "relocate_5pct": relocate,
                           "grow_5pct": grow}, launches, rounds)
    res = {"n_dead": int(dead.sum()), "n_added": u_add.numel()}
    for k, ts in times.items():
        res[k + "_ms"] = round(median(ts), 4)
        res[k + "_ms_rounds"] = [round(t, 4) for t in ts]
    log(f"relocate 5 % dead ({res['n_dead']}): {res['relocate_5pct_ms']:.4f} ms including the opacity restore "
        f"({res['restore_opa_only_ms']:.4f} ms); grow by 5 % ({res['n_added']}): {res['grow_5pct_ms']:.4f} ms")
    del p, m, v
    torch.cuda.empty_cache()
    return res


def bench_step(dev, steps, rounds):
    g = S.make_gaussians(N, W, H, 0, sh_dim=3, opa_range=(0.05, 0.9))
    go = S.make_grad_output(H, W, 0).to(dev)
    legs = {}
    for name in ("plain", "mcmc"):
        sp = splatter.Splatter.from_tensors(g, views_dict(), device=dev, use_sh_coeff=False)
        gs = sp.gaussian_3ds
        opt = optim.FlatAdam([{"params": gs.opa, "lr": 1e-5}, {"params": gs.rgb, "lr": 1e-5},
                              {"params": gs.pos, "lr": 1e-6}, {"params": gs.scale, "lr": 1e-6},
                              {"params": gs.quat, "lr": 1e-6}], betas=BETAS)
        legs[name] = (sp, opt)

    def it(name):
        sp, opt = legs[name]
        opt.zero_grad(set_to_none=True)
        sp(0).backward(go)
        if name == "mcmc":
            sp.add_mcmc_regularizer_grads(0.01, 0.01)
        opt.step()
        if name == "mcmc":
            sp.mcmc_noise(1e-6 * 5e5)

    for name in legs:
        for _ in range(5):
            it(name)
    torch.cuda.synchronize()
    out = {"plain": [], "mcmc": []}
    for _ in range(rounds):
        for key in out:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                it(key)
            e1.record()
            torch.cuda.synchronize()
            out[key].append(e0.elapsed_time(e1) / steps)
    res = {"workload": "C3: 2.4 M Gaussians, 1920x1080, RGB, view 0, forward + backward + FlatAdam"}
    for k, ts in out.items():
        res[k + "_ms"] = round(median(ts), 4)
        res[k + "_ms_rounds"] = [round(t, 4) for t in ts]
    log(f"training step: plain {res['plain_ms']:.4f} ms, with MCMC regulariser + noise {res['mcmc_ms']:.4f} ms")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20, help="timed calls per variant and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-steps", type=int, default=20, help="iterations per round of the training-step leg (0: skip)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    log(f"card: {name}, power limit {limit}")
    gbs, copy_ms = copy_gbs(dev)
    log(f"copy bandwidth {gbs:.0f} GB/s (1 GiB D2D, read + write)")
    res = {"card": name, "power_limit": limit, "N": N,
           "copy": {"bytes": 1 << 30, "ms": round(copy_ms, 4), "GBps": round(gbs, 1)},
           "launches_per_round": args.launches, "rounds": args.rounds,
           "noise": bench_noise(dev, args.launches, args.rounds, gbs),
           "refine": bench_refine(dev, args.launches, args.rounds)}
    if args.e2e_steps > 0:
        res["step"] = bench_step(dev, args.e2e_steps, args.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
