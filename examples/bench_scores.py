"""Cost of the blend-weight score pass (gs_frame_scores) and of pruning by it, on the C3 scene (2.4 M Gaussians,
1920x1080, eight synthetic views), in one process:

  score_1view_ms   one score call after a single-view forward, next to that frame's blend forward and blend
                   backward stage times (gs_frame_stage_ms, frames of their own)
  score_batch8_ms  one score call after a batched forward of the 8 views, per view
  prune_ms         Splatter.prune at 2.4 M keeping the 50 % with the largest weight_sum
  frame_ms         RGB frame forward + backward (Splatter.forward, mean over the 8 views) before and after that prune

Prints the card name and power limit read in the same run, then one JSON line.

  python examples/bench_scores.py [--steps 20] [--rounds 5]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))
sys.path.insert(0, os.path.join(ROOT, "examples"))

import splatter  # noqa: E402
import synthetic as S  # noqa: E402
from bench_surfel import card, median  # noqa: E402

W, H, N, B = 1920, 1080, 2_400_000, 8


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    name, limit = card()
    dev = torch.device("cuda", 0)
    g = S.make_gaussians(N, W, H, 0)
    vs = [S.make_view(W, H, k) for k in range(B)]
    views = [dict(width=v.width, height=v.height, focal_x=v.fx, focal_y=v.fy, rot=v.rot, tran=v.tran) for v in vs]

    def make():
        return splatter.Splatter.from_tensors(g, views, device=dev, near=vs[0].near)

    sp = make()
    sc = splatter.ContributionScores(N, dev)
    gen = torch.Generator().manual_seed(1)
    go = ((torch.rand(H, W, 3, generator=gen) * 2 - 1) / (H * W)).to(dev)
    res = {"card": name, "power_limit": limit, "n": N, "width": W, "height": H, "steps": args.steps,
           "rounds": args.rounds}

    def frame(s, k):
        for p in s.gaussian_3ds.parameters():
            p.grad = None
        s(k).backward(go)

    # stage times of the single-view frame the score pass follows (view 0)
    sp._rctx.set_timing(True)
    stages = []
    for _ in range(args.rounds + 1):
        frame(sp, 0)
        stages.append(sp._rctx.stage_ms())
    sp._rctx.set_timing(False)
    stages = stages[1:]
    res["blend_fwd_ms"] = round(median([x[5] for x in stages]), 4)
    res["blend_bwd_ms"] = round(median([x[6] for x in stages]), 4)
    st = sp.frame_stats()
    res["M"], res["M_eff"] = st["n_instances"], st["n_instances_eff"]

    one, batch = [], []
    for _ in range(args.rounds):
        with torch.no_grad():
            sp(0)
        sp.accumulate_scores(sc)                               # warm-up and workspace growth
        one.append(timed(lambda: sp.accumulate_scores(sc), args.steps))
        with torch.no_grad():
            sp.render_batch(range(B))
        sp.accumulate_scores(sc)
        batch.append(timed(lambda: sp.accumulate_scores(sc), args.steps) / B)
    res["score_1view_ms"] = round(median(one), 4)
    res["score_batch8_ms_per_view"] = round(median(batch), 4)

    def frames(s):
        for k in range(B):
            frame(s, k)
        return timed(lambda: [frame(s, k) for k in range(B)], max(1, args.steps // B)) / B

    before = [frames(sp) for _ in range(args.rounds)]
    scores = sp.score_views(batch_size=B)
    keep = torch.zeros(N, dtype=torch.bool, device=dev).index_fill_(
        0, torch.sort(scores.weight_sum, descending=True, stable=True).indices[:N // 2], True)
    prune = []
    for _ in range(args.rounds):
        s2 = make()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        s2.prune(keep)
        e1.record()
        torch.cuda.synchronize()
        prune.append(e0.elapsed_time(e1))
        del s2
    res["prune_ms"] = round(median(prune), 4)
    sp.prune(keep)
    after = [frames(sp) for _ in range(args.rounds)]
    res["frame_ms_before"] = round(median(before), 4)
    res["frame_ms_after"] = round(median(after), 4)
    res["n_after"] = sp.gaussian_3ds.pos.shape[0]
    res["weight_sum_kept_share"] = round(float(scores.weight_sum[keep].double().sum() /
                                               scores.weight_sum.double().sum()), 6)
    print(f"card: {name}, power limit {limit}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
