"""Per-view camera pose gradients of a batched frame (renderer.render_frame_batch_cam) against the same views
differentiated one after another with renderer.render_frame_cam (the frame Splatter.render_at_pose runs), on the C3
scene (2.4 M Gaussians) at 1920x1080 and, zoomed out, at 480x270 (the bench_batch.py views).

For RGB colour and per-Gaussian SH of degree 3, and B = 1, 2, 4, 8 views at orbit poses k * 45 deg (and B = 64 at
480x270, where the per-view CTA sums of the camera gradient add up), it times per view:
  seq_full:   B single-view camera frames, forward + backward, gradients of the five parameters and of the pose;
  batch_full: one frame of B views and its backward, the same gradients;
  seq_cam / batch_cam: the same, camera only (the scene frozen: pose tracking, multi-hypothesis localisation).
The four are alternated in one process (5 rounds of 10 steps by default; medians).  A separate pass reads the
projection-backward stage (stage 7 of gs_frame_stage_ms: the projection backward, plus the camera finishing sums where
they run) of render_frame_batch and of render_frame_batch_cam with parameter gradients.  Prints the card name and
power limit read in the same run, then one JSON line.

  python examples/bench_batch_pose.py [--steps 10] [--rounds 5]
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
RUNS = [((1920, 1080), (1, 2, 4, 8)), ((480, 270), (1, 2, 4, 8, 64))]
PROJECT_BWD = 7   # gs_frame_stage_ms index of the projection backward


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
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--n", type=int, default=2_400_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    scenes, frozen, rctxs = {}, {}, {}
    for colour, sh_dim in (("rgb", 3), ("sh48", 48)):
        g = S.make_gaussians(args.n, 1920, 1080, 0, sh_dim)
        scenes[colour] = {k: t.to(dev).requires_grad_(True) for k, t in g.items()}
        frozen[colour] = {k: t.detach() for k, t in scenes[colour].items()}
        rctx = gaussian.RenderContext()
        if colour != "rgb":
            rctx.set_sh_eval(renderer.SH_EVAL["gaussian"])
        rctxs[colour] = rctx

    variants = {}
    for (w, h), batches in RUNS:
        views = [S.make_view(w, h, k % 8) for k in range(max(batches))]
        for colour in scenes:
            for b in batches:
                vs = views[:b]
                go = ((torch.rand(b, h, w, 3, generator=torch.Generator().manual_seed(1)) * 2 - 1) / (h * w)).to(dev)
                rot = torch.stack([v.rot for v in vs]).to(dev)
                tran = torch.stack([v.tran for v in vs]).to(dev)
                variants[f"{w}x{h}_{colour}_B{b}"] = (colour, w, h, vs, go, rot, tran)

    def params(colour, full):
        p = scenes[colour] if full else frozen[colour]
        if full:
            for t in p.values():
                t.grad = None
        return p

    def sequential(label, full):
        colour, w, h, vs, go, rot, tran = variants[label]
        p = params(colour, full)
        for k, v in enumerate(vs):
            r, t = rot[k].clone().requires_grad_(True), tran[k].clone().requires_grad_(True)
            img, _, _, _ = renderer.render_frame_cam(rctxs[colour], *(p[q] for q in NAMES), w, h, v.fx, v.fy, r, t,
                                                     v.near, 0.05, "abs")
            img.backward(go[k])

    def batched(label, full, cam=True):
        colour, w, h, vs, go, rot, tran = variants[label]
        p = params(colour, full)
        r, t = rot.clone().requires_grad_(cam), tran.clone().requires_grad_(cam)
        fn = renderer.render_frame_batch_cam if cam else renderer.render_frame_batch
        img, _, _, _ = fn(rctxs[colour], *(p[q] for q in NAMES), w, h, [v.fx for v in vs], [v.fy for v in vs], r, t,
                          vs[0].near, 0.05, "abs")
        img.backward(go)

    modes = {"seq_full": lambda lb: sequential(lb, True), "batch_full": lambda lb: batched(lb, True),
             "seq_cam": lambda lb: sequential(lb, False), "batch_cam": lambda lb: batched(lb, False)}
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

    # stage 7 (projection backward) of the plain batched frame and of the camera-gradient batched frame, alternated
    for rctx in rctxs.values():
        rctx.set_timing(True)
    stage = {(label, m): [] for label in variants for m in ("batch", "batch_cam")}
    for _ in range(args.rounds):
        for label, var in variants.items():
            for m in ("batch", "batch_cam"):
                batched(label, True, cam=m == "batch_cam")
                stage[(label, m)].append(rctxs[var[0]].stage_ms()[PROJECT_BWD])
    for rctx in rctxs.values():
        rctx.set_timing(False)

    res = {"card": name, "power_limit": limit, "n": args.n, "steps": args.steps, "rounds": args.rounds,
           "workload": "C3 scene, forward + backward, upstream image gradient only; ms per view"}
    for label in variants:
        r = {}
        for m in modes:
            r[f"{m}_ms_per_view"] = round(median(times[(label, m)]), 4)
            r[f"{m}_ms_all"] = [round(t, 4) for t in times[(label, m)]]
        r["full_batch_over_seq"] = round(r["batch_full_ms_per_view"] / r["seq_full_ms_per_view"], 4)
        r["cam_batch_over_seq"] = round(r["batch_cam_ms_per_view"] / r["seq_cam_ms_per_view"], 4)
        r["stage7_batch_ms"] = round(median(stage[(label, "batch")]), 4)
        r["stage7_batch_cam_ms"] = round(median(stage[(label, "batch_cam")]), 4)
        res[label] = r
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
