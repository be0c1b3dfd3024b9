#!/usr/bin/env python
"""Run the reference's `train.py` UNCHANGED on this framework, on 1..8 GPUs (SURVEY.md §8 f-1,
"8 views sharded across 8 GPUs, NCCL grad allreduce, train.py loop").

    python dp_launch.py [--train-py PATH] [--splatter ours|reference] [--torch-adam] -- <train.py arguments>
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 dp_launch.py -- --data ...

Nothing in train.py is edited; this launcher only arranges what surrounds it:

* `sys.path`: `shims/` (torchmetrics / kornia / pykdtree / viser / omegaconf stand-ins, see shims/README.md),
  then this package (`gaussian` extension, `renderer`, `splatter`, `loss`), then the directory of train.py
  (its own `utils.py`, `visergui.py`).  `--splatter reference` keeps the reference's splatter.py /
  renderer.py as well, so that only the `gaussian` extension module is ours (legacy per-stage boundary).
* one process per GPU (torchrun env): NCCL group, `cuda:LOCAL_RANK` current; numpy seeded PER RANK
  (`--seed base + rank`: train.py:93 draws the camera with numpy, so each rank renders a different view),
  torch seeded IDENTICALLY (densification samples split positions with torch: replicas must stay equal).
* the gradient exchange, placed between `loss.backward()` and `optimizer.step()` (train.py:118-120)
  by giving `torch.optim.Adam` a `step()` that first averages the flat gradient bucket over the ranks
  (`dp.make_grad_bucket`: NVLink push / peer kernels or one NCCL all-reduce); by default the update itself is
  the fused flat Adam (`optim.FlatAdam`, csrc/optim.cu), `--torch-adam` keeps torch's.
* densification statistics that are per-view in the reference (train.py:148-150): `Splatter.culling_mask`
  is summed over ranks after every training forward, `pos.grad` is already the exchanged gradient - every
  replica takes identical prune / clone / split decisions.
* ranks > 0 write their images / checkpoints to `<exp>_rank<r>` (identical content, no clobbering).
"""
from __future__ import annotations

import argparse
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _parse(argv):
    if "--" in argv:
        k = argv.index("--")
        own, rest = argv[:k], argv[k + 1:]
    else:
        own, rest = [], argv
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--train-py", default=os.environ.get("GS_TRAIN_PY", os.path.join(os.getcwd(), "train.py")),
                    help="path of the reference's train.py (default: $GS_TRAIN_PY, else ./train.py)")
    ap.add_argument("--splatter", default="ours", choices=["ours", "reference"])
    ap.add_argument("--torch-adam", action="store_true", help="keep torch.optim.Adam's update (default: fused FlatAdam)")
    ap.add_argument("--torch-seed", type=int, default=1234)
    return ap.parse_args(own), rest


def _get_opt(args, name, default):
    if name in args:
        return args[args.index(name) + 1]
    return default


def _set_opt(args, name, value):
    if name in args:
        args[args.index(name) + 1] = str(value)
    else:
        args += [name, str(value)]


def main():
    own, targv = _parse(sys.argv[1:])
    train_py = os.path.abspath(own.train_py)
    if not os.path.exists(train_py):
        raise SystemExit(f"train.py not found at {train_py} (pass --train-py)")
    ref_dir = os.path.dirname(train_py)
    paths = [os.path.join(ROOT, "shims"), HERE, ref_dir]
    sys.path[:0] = paths

    import torch
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        _set_opt(targv, "--seed", int(_get_opt(targv, "--seed", 2023)) + rank)     # train.py:332,364
        if rank > 0:
            _set_opt(targv, "--exp", f"{_get_opt(targv, '--exp', 'default')}_rank{rank}")
    torch.manual_seed(own.torch_seed)                       # identical on every rank (utils.py:391-402)

    import gaussian  # noqa: F401  ours; must be imported before anything binds the name
    if own.splatter == "reference":
        # the reference's splatter.py + renderer.py on OUR extension module: load them under their own names
        import importlib.util
        for name in ("renderer", "splatter"):
            spec = importlib.util.spec_from_file_location(name, os.path.join(ref_dir, name + ".py"))
            mod = importlib.util.module_from_spec(spec)
            sys.modules[name] = mod
            spec.loader.exec_module(mod)
    import dp
    import splatter

    base_adam = torch.optim.Adam
    if not own.torch_adam and own.splatter == "ours":
        import optim
        base_adam = optim.FlatAdam

    class DPAdam(base_adam):
        """torch.optim.Adam as train.py constructs it (train.py:56-64,173-181) + the gradient exchange."""

        def __init__(self, params, **kw):
            super().__init__(params, **kw)
            ps = [p for g in self.param_groups for p in g["params"]]
            # the fused backward lays its gradients out in (pos, rgb, opa, quat, scale) order
            g3 = {id(p): p for p in ps}
            self._bucket = dp.make_grad_bucket(list(g3.values()), average=True) if world > 1 else None
            self._order = None

        def step(self, closure=None):
            if self._bucket is not None:
                if self._order is None:              # bucket order = memory order of the flat gradient buffer
                    ps = [p for g in self.param_groups for p in g["params"] if p.grad is not None]
                    ps.sort(key=lambda p: p.grad.data_ptr())
                    self._bucket.params = ps
                    self._order = True
                self._bucket.allreduce()
            return super().step() if closure is None else super().step(closure)

    torch.optim.Adam = DPAdam

    if world > 1:
        fwd = splatter.Splatter.forward

        def forward(self, *a, **k):
            out = fwd(self, *a, **k)
            if torch.is_grad_enabled() and getattr(self, "culling_mask", None) is not None:
                m = self.culling_mask.clone()
                dist.all_reduce(m)                   # train.py:150: visibility counts over all ranks' views
                self.culling_mask = m
            return out

        splatter.Splatter.forward = forward

    sys.argv = [train_py] + targv
    try:
        runpy.run_path(train_py, run_name="__main__")
    finally:
        if world > 1 and dist.is_initialized():
            dist.barrier()
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
