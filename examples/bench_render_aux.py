"""Cost of the depth / alpha maps and the background colour on the C3 frame (2.4 M Gaussians, 1080p).

For each colour width D = 3 (RGB), 27 and 48 (per-pixel SH, default kernels) it times forward + backward of one
frame in three configurations, alternating them in one process so that they share the card's state:  plain
(render_frame_final), background only (render_frame_aux with a background, image gradient only: plain backward
kernels), aux (depth and alpha gradients too: the aux backward kernels).  Prints the card name and power limit
read in the same run, then one JSON line.

  python examples/bench_render_aux.py [--steps 20] [--rounds 5] [--colours 3,27,48]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

import renderer  # noqa: E402
import synthetic as S  # noqa: E402
import gaussian  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in out.split(","))
    except Exception:  # noqa: BLE001 - report what torch knows
        name, limit = torch.cuda.get_device_name(0), "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--colours", default="3,27,48")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    res = {"card": name, "power_limit": limit, "workload": "C3 forward+backward", "steps": args.steps,
           "rounds": args.rounds}
    for d in (int(c) for c in args.colours.split(",")):
        res[f"D{d}"] = bench_colour(d, args.steps, args.rounds)
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


def bench_colour(d, steps, rounds):
    dev = torch.device("cuda", 0)
    n, w, h = 2_400_000, 1920, 1080
    g = {k: t.to(dev) for k, t in S.make_gaussians(n, w, h, 0, sh_dim=d).items()}
    v = S.make_view(w, h, 0)
    cam = (w, h, v.fx, v.fy, v.rot, v.tran, v.near, 0.05, "abs")
    gen = torch.Generator().manual_seed(1)
    go = ((torch.rand(h, w, 3, generator=gen) * 2 - 1) / (h * w)).to(dev)
    gd = ((torch.rand(h, w, generator=gen) * 2 - 1) / (h * w)).to(dev)
    ga = ((torch.rand(h, w, generator=gen) * 2 - 1) / (h * w)).to(dev)
    params = {k: t.clone().requires_grad_(True) for k, t in g.items()}
    rctx = gaussian.RenderContext()
    bg = (1.0, 1.0, 1.0)

    def plain():
        img, _ = renderer.render_frame_final(rctx, *(params[k] for k in ("pos", "rgb", "opa", "quat", "scale")), *cam)
        img.backward(go)

    def background():
        img, _, _, _ = renderer.render_frame_aux(rctx, *(params[k] for k in ("pos", "rgb", "opa", "quat", "scale")),
                                                 *cam, background=bg)
        img.backward(go)

    def aux():
        img, dep, alp, _ = renderer.render_frame_aux(rctx, *(params[k] for k in ("pos", "rgb", "opa", "quat", "scale")),
                                                     *cam, background=bg)
        torch.autograd.backward([img, dep, alp], [go, gd, ga])

    variants = {"plain": plain, "background": background, "aux": aux}
    for fn in variants.values():          # warm-up: module loads, workspace growth
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(rounds):
        for name, fn in variants.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                for p in params.values():
                    p.grad = None
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / steps)
    res = {}
    for k, ts in times.items():
        res[f"{k}_ms_median"] = sorted(ts)[len(ts) // 2]
        res[f"{k}_ms_all"] = [round(t, 4) for t in ts]
    res["background_over_plain"] = res["background_ms_median"] / res["plain_ms_median"]
    res["aux_over_plain"] = res["aux_ms_median"] / res["plain_ms_median"]
    return res


if __name__ == "__main__":
    main()
