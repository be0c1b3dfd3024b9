"""The optimizer step at C3 size (2.4 M Gaussians): dense fused Adam (gs_adam_step) against visible-only Adam
(gs_adam_step_visible) for the three colour widths (RGB D = 3, per-Gaussian SH degree 2 D = 27, degree 3 D = 48).

In one process, on the GPU (no device: it fails, there is no fallback):
  * a 1 GiB device-to-device copy timed with CUDA events: the HBM bandwidth this card reaches (read + written bytes);
  * the visibility masks of real frames: bench.py's C3 scene (seed 0, 1920x1080) rendered at view 0, as one
    `render_batch` of 8 views, and at a close-up (view 0 at twice the focal length); their visible fractions are
    printed;
  * per D: flat buffers in the bucket's layout filled from a seed; the dense kernel and the visible-only kernel at
    f in {1, 0.5, 0.25, 0.1} with a uniformly random mask and with a mask of contiguous runs, and with the real
    masks.  Variants are alternated inside every round; a round times --launches launches per variant between two
    CUDA events; the figure is the median of --rounds rounds (>= 200 timed launches per variant by default);
  * algorithmic bytes 28 (11 + D) N_vis + N (four streams read, three written per visible float, plus the mask), the
    rate they give, and that rate's share of the copy's;
  * end to end: frame (forward + backward, per-Gaussian SH degree 3) + optimizer step per iteration through Splatter
    and FlatAdam, dense against visible-only, at view 0 and at the close-up.
The card's name and power limit are read (query only) and printed with the numbers.  Human-readable lines go to
stderr, one JSON line to stdout.

  python examples/bench_optim.py [--launches 50] [--rounds 5] [--e2e-steps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

import gaussian  # noqa: E402
import optim  # noqa: E402
import splatter  # noqa: E402
import synthetic as S  # noqa: E402

N, W, H = 2_400_000, 1920, 1080
BETAS, EPS = (0.9, 0.99), 1e-8
FRACTIONS = (1.0, 0.5, 0.25, 0.1)
RUN = 4096                      # rows per run of the run-structured masks


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
    except Exception:  # noqa: BLE001 - report what torch knows
        name, limit = torch.cuda.get_device_name(0), "unknown"
    return name, limit


def median(ts):
    return sorted(ts)[len(ts) // 2]


def copy_gbs(dev, nbytes=1 << 30, iters=20):
    """Device-to-device copy of nbytes: (read + written bytes) / time, median of iters timed copies."""
    src = torch.empty(nbytes // 4, dtype=torch.float32, device=dev).uniform_()
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = median(ts)
    del src, dst
    torch.cuda.empty_cache()
    return 2 * nbytes / (ms * 1e-3) / 1e9, ms


def layout(n, d):
    """The gradient bucket's layout (renderer._flat_grads): pos 3, rgb d, opa 1, quat 4, scale 3, each padded to 4."""
    widths = [3, d, 1, 4, 3]
    starts, o = [], 0
    for w in widths:
        starts.append(o)
        o += (n * w + 3) // 4 * 4
    return starts, widths, o


def synthetic_masks(n, dev):
    gen = torch.Generator().manual_seed(0)
    out = {}
    for f in FRACTIONS:
        if f == 1.0:
            out[("all", f)] = torch.ones(n, dtype=torch.uint8, device=dev)
            continue
        out[("random", f)] = (torch.rand(n, generator=gen) < f).to(torch.uint8).to(dev)
        k = (n + RUN - 1) // RUN
        on = torch.zeros(k, dtype=torch.bool)
        on[torch.randperm(k, generator=gen)[:round(f * k)]] = True
        out[("runs", f)] = on.repeat_interleave(RUN)[:n].to(torch.uint8).to(dev)
    return out


CLOSE_UP = 8                    # index of the close-up view in views_dict()


def views_dict():
    """bench.py's 8 views, which all contain the whole synthetic scene, and view 0 again at twice its focal length:
    a close-up that leaves most of the scene outside the image, as a training view of a captured scene does."""
    views = [S.make_view(W, H, k) for k in range(8)]
    vd = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in views]
    return vd + [dict(vd[0], focal_x=2 * vd[0]["focal_x"], focal_y=2 * vd[0]["focal_y"])]


def real_masks(dev):
    """Masks of bench.py's C3 scene: view 0, the 8 views as one batch, and the close-up.  Visibility does not depend
    on the colour model, so the RGB scene stands for all three widths."""
    g = S.make_gaussians(N, W, H, 0, sh_dim=3, opa_range=(0.05, 0.9))
    sp = splatter.Splatter.from_tensors(g, views_dict(), device=dev, use_sh_coeff=False)
    with torch.no_grad():
        sp(0)
        one = sp.visible_mask().clone()
        sp.render_batch(list(range(8)))
        batch = sp.visible_mask().clone()
        sp(CLOSE_UP)
        close = sp.visible_mask().clone()
    torch.cuda.synchronize()
    del sp
    torch.cuda.empty_cache()
    return {(k, float(m.float().mean())): m for k, m in (("view0", one), ("batch8", batch), ("closeup", close))}


def time_variants(variants, launches, rounds):
    """{name: [ms per launch, one per round]}; every round runs every variant once, in the same order."""
    for fn in variants.values():                      # module load, first touch
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    out = {k: [] for k in variants}
    for _ in range(rounds):
        for k, fn in variants.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                fn()
            e1.record()
            torch.cuda.synchronize()
            out[k].append(e0.elapsed_time(e1) / launches)
    return out


def bench_width(d, masks, dev, launches, rounds, gbs):
    starts, widths, total = layout(N, d)
    ends = starts[1:] + [total]
    lrs = [0.003, 0.03, 0.03, 0.003, 0.003]
    gen = torch.Generator(device=dev).manual_seed(d)
    p, g = (torch.randn(total, generator=gen, device=dev) for _ in range(2))
    g *= 1e-3
    m, v = torch.zeros_like(p), torch.zeros_like(p)

    variants = {"dense": lambda: gaussian.adam_step(p, g, m, v, ends, lrs, *BETAS, EPS, 10)}
    for key, mask in masks.items():
        variants[key] = (lambda mk: lambda: gaussian.adam_step_visible(p, g, m, v, starts, widths, lrs, mk, *BETAS,
                                                                       EPS, 10))(mask)
    times = time_variants(variants, launches, rounds)
    dense_ms = median(times["dense"])
    rows = []
    for key, ts in times.items():
        ms = median(ts)
        if key == "dense":
            kind, f, n_vis, nbytes = "dense", 1.0, N, 28 * total
        else:
            kind, f = key
            n_vis = int(masks[key].sum())
            nbytes = 28 * (11 + d) * n_vis + N
        rate = nbytes / (ms * 1e-3) / 1e9
        rows.append({"D": d, "kernel": "dense" if key == "dense" else "visible", "mask": kind, "f": round(f, 4),
                     "n_visible": n_vis, "ms": round(ms, 4), "ms_rounds": [round(t, 4) for t in ts],
                     "MB": round(nbytes / 1e6, 1), "GBps": round(rate, 1), "share_of_copy": round(rate / gbs, 3),
                     "vs_dense": round(ms / dense_ms, 3)})
        log(f"D={d:<3} {rows[-1]['kernel']:<8} {kind:<7} f={f:6.3f}  {ms:8.4f} ms  {nbytes / 1e6:8.1f} MB "
            f"{rate:7.0f} GB/s  {rate / gbs:6.1%} of copy   x{ms / dense_ms:5.3f} of dense")
    del p, g, m, v
    torch.cuda.empty_cache()
    return rows


def bench_e2e(dev, steps, rounds, view):
    """Frame + optimizer step, per-Gaussian SH degree 3, one view: dense against visible-only, alternated by round."""
    g = S.make_gaussians(N, W, H, 0, sh_dim=48, opa_range=(0.05, 0.9))
    go = S.make_grad_output(H, W, 0).to(dev)
    legs = {}
    for name in ("dense", "visible"):
        sp = splatter.Splatter.from_tensors(g, views_dict(), device=dev, use_sh_coeff=True, sh_eval="gaussian")
        gs = sp.gaussian_3ds
        opt = optim.FlatAdam([{"params": gs.opa, "lr": 1e-5}, {"params": gs.rgb, "lr": 1e-5},
                              {"params": gs.pos, "lr": 1e-6}, {"params": gs.scale, "lr": 1e-6},
                              {"params": gs.quat, "lr": 1e-6}], betas=BETAS)
        legs[name] = (sp, opt)

    def it(name):
        sp, opt = legs[name]
        opt.zero_grad(set_to_none=True)
        sp(view).backward(go)
        if name == "visible":
            opt.step(visible=sp.visible_mask())
        else:
            opt.step()

    def frame_only(name):
        sp, opt = legs[name]
        opt.zero_grad(set_to_none=True)
        sp(view).backward(go)

    for name in legs:
        for _ in range(5):
            it(name)
    torch.cuda.synchronize()
    out = {"dense": [], "visible": [], "frame_only": []}
    for _ in range(rounds):
        for key, fn in (("dense", lambda: it("dense")), ("visible", lambda: it("visible")),
                        ("frame_only", lambda: frame_only("dense"))):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            out[key].append(e0.elapsed_time(e1) / steps)
    f = float(legs["visible"][0].visible_mask().float().mean())
    res = {"workload": f"C3: 2.4 M Gaussians, 1920x1080, per-Gaussian SH degree 3, "
                       f"{'close-up of view 0' if view == CLOSE_UP else f'view {view}'}, forward + backward + Adam",
           "visible_fraction": round(f, 4)}
    for k, ts in out.items():
        res[k + "_ms"] = round(median(ts), 4)
        res[k + "_ms_rounds"] = [round(t, 4) for t in ts]
    log(f"end to end (SH degree 3, view {view}, visible fraction {f:.3f}): frame only {res['frame_only_ms']:.4f} ms, "
        f"frame + dense Adam {res['dense_ms']:.4f} ms, frame + visible-only Adam {res['visible_ms']:.4f} ms")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50, help="timed launches per variant and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-steps", type=int, default=20, help="iterations per round of the end-to-end leg (0: skip)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    log(f"card: {name}, power limit {limit}")
    gbs, copy_ms = copy_gbs(dev)
    log(f"copy bandwidth {gbs:.0f} GB/s (1 GiB D2D, read + write)")
    masks = synthetic_masks(N, dev)
    real = real_masks(dev)
    for (kind, f) in real:
        log(f"real mask {kind}: visible fraction {f:.4f}")
    masks.update(real)
    res = {"card": name, "power_limit": limit, "N": N,
           "copy": {"bytes": 1 << 30, "ms": round(copy_ms, 4), "GBps": round(gbs, 1)},
           "launches_per_round": args.launches, "rounds": args.rounds,
           "real_visible_fraction": {kind: round(f, 4) for (kind, f) in real}, "kernels": []}
    for d in (3, 27, 48):
        res["kernels"] += bench_width(d, masks, dev, args.launches, args.rounds, gbs)
    if args.e2e_steps > 0:
        res["end_to_end"] = [bench_e2e(dev, args.e2e_steps, args.rounds, view) for view in (0, CLOSE_UP)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
