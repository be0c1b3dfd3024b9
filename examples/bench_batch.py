"""Batched frames (renderer.render_frame_batch) against the same views rendered one after another, on the C3 scene
(2.4 M Gaussians) at 1920x1080 and, zoomed out, at 480x270 (the same scene, a quarter of the focal length: the
bench_filter.py view).

For RGB colour and per-Gaussian SH of degree 3, and B = 1, 2, 4, 8 views at orbit poses k * 45 deg, it times per view:
  sequential: B single-view frames (render_frame_aux, forward + backward, the gradients accumulated into .grad by
              autograd), the training loop without batching;
  batched:    one frame of B views and its backward.
The two are alternated in one process (5 rounds of 20 steps by default; medians).  A separate pass reads the per-stage
device times (CUDA events; the sequential ones summed over its B frames) and M / M_eff.  Prints the card name and power
limit read in the same run, then one JSON line.

  python examples/bench_batch.py [--steps 20] [--rounds 5]
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

NAMES = ("pos", "rgb", "opa", "quat", "scale")
SIZES = ((1920, 1080), (480, 270))
BATCHES = (1, 2, 4, 8)
# gs_frame_stage_ms indices
STAGES = {"project_fwd": 0, "sort_scan": 1, "emit": 2, "tile_sort": 3, "ranges": 4, "blend_fwd": 5, "blend_bwd": 6,
          "project_bwd": 7}


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--n", type=int, default=2_400_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    scenes = {}
    for colour, sh_dim in (("rgb", 3), ("sh48", 48)):
        g = S.make_gaussians(args.n, 1920, 1080, 0, sh_dim)
        scenes[colour] = {k: t.to(dev).requires_grad_(True) for k, t in g.items()}
    rctxs = {}
    for colour in scenes:
        rctx = gaussian.RenderContext()
        if colour != "rgb":
            rctx.set_sh_eval(renderer.SH_EVAL["gaussian"])
        rctxs[colour] = rctx

    variants = {}
    for w, h in SIZES:
        views = [S.make_view(w, h, k) for k in range(max(BATCHES))]
        for colour in scenes:
            for b in BATCHES:
                vs = views[:b]
                go = ((torch.rand(b, h, w, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) / (h * w)).to(dev)
                variants[f"{w}x{h}_{colour}_B{b}"] = (colour, w, h, vs, go)

    def sequential(label):
        colour, w, h, vs, go = variants[label]
        p, rctx = scenes[colour], rctxs[colour]
        for t in p.values():
            t.grad = None
        for k, v in enumerate(vs):
            img, _, _, _ = renderer.render_frame_aux(rctx, *(p[q] for q in NAMES), w, h, v.fx, v.fy, v.rot, v.tran,
                                                     v.near, 0.05, "abs")
            img.backward(go[k])

    def batched(label):
        colour, w, h, vs, go = variants[label]
        p, rctx = scenes[colour], rctxs[colour]
        for t in p.values():
            t.grad = None
        img, _, _, _ = renderer.render_frame_batch(rctx, *(p[q] for q in NAMES), w, h, [v.fx for v in vs],
                                                   [v.fy for v in vs], torch.stack([v.rot for v in vs]),
                                                   torch.stack([v.tran for v in vs]), vs[0].near, 0.05, "abs")
        img.backward(go)

    modes = {"sequential": sequential, "batched": batched}
    for label in variants:                 # warm-up: module loads, workspace growth
        for fn in modes.values():
            for _ in range(2):
                fn(label)
    torch.cuda.synchronize()
    times = {(label, m): [] for label in variants for m in modes}
    for _ in range(args.rounds):
        for label in variants:
            for m, fn in modes.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.steps):
                    fn(label)
                e1.record()
                torch.cuda.synchronize()
                times[(label, m)].append(e0.elapsed_time(e1) / args.steps / len(variants[label][3]))

    # per-stage device times and instance counts, one frame per round (sequential: summed over its B frames)
    for rctx in rctxs.values():
        rctx.set_timing(True)
    stages = {(label, m): {s: [] for s in STAGES} for label in variants for m in modes}
    counts = {}
    for _ in range(args.rounds):
        for label, (colour, w, h, vs, go) in variants.items():
            rctx = rctxs[colour]
            for m in modes:
                tot = {s: 0.0 for s in STAGES}
                if m == "batched":
                    batched(label)
                    ms = rctx.stage_ms()
                    for s, i in STAGES.items():
                        tot[s] = ms[i]
                    st = rctx.stats()
                    counts[label] = (st["n_instances"], st["n_instances_eff"])
                else:
                    p = scenes[colour]
                    for k, v in enumerate(vs):
                        img, _, _, _ = renderer.render_frame_aux(rctx, *(p[q] for q in NAMES), w, h, v.fx, v.fy,
                                                                 v.rot, v.tran, v.near, 0.05, "abs")
                        img.backward(go[k])
                        ms = rctx.stage_ms()
                        for s, i in STAGES.items():
                            tot[s] += ms[i]
                for s in STAGES:
                    stages[(label, m)][s].append(tot[s])
    for rctx in rctxs.values():
        rctx.set_timing(False)

    res = {"card": name, "power_limit": limit, "n": args.n, "steps": args.steps, "rounds": args.rounds,
           "workload": "C3 scene, forward + backward, upstream image gradient only; ms per view"}
    for label in variants:
        r = {}
        for m in modes:
            r[f"{m}_ms_per_view"] = round(median(times[(label, m)]), 4)
            r[f"{m}_ms_all"] = [round(t, 4) for t in times[(label, m)]]
            r[f"{m}_stage_ms"] = {s: round(median(v), 4) for s, v in stages[(label, m)].items()}
        r["batched_over_sequential"] = round(r["batched_ms_per_view"] / r["sequential_ms_per_view"], 4)
        r["n_instances"], r["n_instances_eff"] = counts[label]
        res[label] = r
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
