"""Checkpoints (SURVEY.md §8 f-4).

`save_checkpoint` writes the reference's key schema (train.py:283-291: a dict with the five parameter
tensors `pos, opa, rgb, quat, scale`, so the reference's own `--ckpt` / `Splatter(load_ckpt=...)` path,
splatter.py:417-424, loads our files and we load theirs) and - what the reference lacks - everything a
true resume needs under the extra key `"resume"`: optimizer moments and step count, iteration, the
densification statistics of train.py:82-83, and the RNG states (numpy picks the camera, train.py:93;
torch samples split positions, utils.py:391-402).  A scene with per-Gaussian features
(`Splatter(..., n_features=F)`) also stores them under `"feat"` [n, F].  Extra keys are ignored by the reference's
loader.  A scene with Mip-Splatting's 3-D filter (`Splatter(..., filter3d=True)`) stores the filter under
`"filter3d"` [n], so that a resume renders the same bits; loading a file without it recomputes the filter.  Per-view
bilateral grids (`bilagrid.BilateralGrids`) and their optimizer go under `"bilagrid"` (`grids` and the optimizer's
state dict), so that a resume restores the grids and their Adam moments.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

KEYS = ("pos", "opa", "rgb", "quat", "scale")          # train.py:284-290 order


def _optimizer_state(opt):
    if opt is None:
        return None
    if hasattr(opt, "state_dict"):
        return {"kind": "torch", "state": opt.state_dict()}
    # optim.FlatAdam: flat moments + per-group learning rates
    flat = getattr(opt, "_flat", None)
    staged = getattr(opt, "_staged", None)     # moments carried over a growth (FlatAdam.replace_params), not yet placed
    return {"kind": "flat_adam", "step": opt.step_count, "betas": opt.betas, "eps": opt.eps,
            "lrs": [g["lr"] for g in opt.param_groups],
            "exp_avg": None if flat is None else flat[1].detach().cpu(),
            "exp_avg_sq": None if flat is None else flat[2].detach().cpu(),
            "staged": None if staged is None else [None if s is None else (s[0].detach().cpu(), s[1].detach().cpu())
                                                   for s in staged]}


def save_checkpoint(splatter, path, optimizer=None, iteration: Optional[int] = None, trainer_state: Optional[dict] = None,
                    bilagrid=None, bilagrid_optimizer=None):
    """`path` is the checkpoint file (train.py writes `<exp>/ckpt.pth`)."""
    g = splatter.gaussian_3ds
    ckpt = {k: getattr(g, k).detach().clone() for k in KEYS}
    if g.feat is not None:
        ckpt["feat"] = g.feat.detach().clone()
    if getattr(splatter, "filter3d", None) is not None:
        ckpt["filter3d"] = splatter.filter3d.detach().clone()
    if bilagrid is not None:
        ckpt["bilagrid"] = {"grids": bilagrid.grids.detach().cpu().clone(),
                            "optimizer": None if bilagrid_optimizer is None else bilagrid_optimizer.state_dict()}
    ckpt["resume"] = {
        "iteration": iteration,
        "optimizer": _optimizer_state(optimizer),
        "trainer": {k: (v.detach().cpu() if torch.is_tensor(v) else v) for k, v in (trainer_state or {}).items()},
        "torch_rng": torch.get_rng_state(),
        "cuda_rng": torch.cuda.get_rng_state(splatter.device) if torch.cuda.is_available() else None,
        "numpy_rng": np.random.get_state(),
        "scale_activation": splatter.scale_activation,
        "use_sh_coeff": splatter.use_sh_coeff,
    }
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    tmp = path + ".tmp"
    torch.save(ckpt, tmp)
    os.replace(tmp, path)                                   # a crash never leaves a truncated checkpoint
    return path


def load_checkpoint(path, splatter=None, optimizer=None, restore_rng=True, bilagrid=None, bilagrid_optimizer=None):
    """Returns the dict; with `splatter` the parameters are replaced in place (new nn.Parameters, like
    adaptive_control - rebuild torch optimizers before passing them here), the features too when the file has them
    (a splatter with features loading a file without them gets zero features); with `optimizer` its state is restored.
    A reference-written file (five keys only) loads the parameters and returns `resume == None`.  With `bilagrid` (a
    BilateralGrids of the saved shape) the grids are copied into its Parameter in place, so optimizers over it stay
    valid, and `bilagrid_optimizer` gets their saved state; a file without grids leaves both as they are."""
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    missing = [k for k in KEYS if k not in ckpt]
    if missing:
        raise KeyError(f"{path}: not a checkpoint of this family, missing {missing}")
    res = ckpt.get("resume")
    if splatter is not None:
        g = splatter.gaussian_3ds
        with torch.no_grad():
            for k in KEYS:
                t = ckpt[k].detach().to(device=splatter.device, dtype=torch.float32).contiguous()
                setattr(g, k, torch.nn.Parameter(t))
            n = g.pos.shape[0]
            if ckpt.get("feat") is not None:
                f = ckpt["feat"].detach().to(device=splatter.device, dtype=torch.float32).contiguous()
                if f.shape[0] != n or (splatter.n_features and f.shape[1] != splatter.n_features):
                    raise ValueError(f"{path}: feat {list(f.shape)} does not fit {n} Gaussians with "
                                     f"{splatter.n_features} features")
                g.feat = torch.nn.Parameter(f)
                splatter.n_features = int(f.shape[1])
            elif g.feat is not None:
                g.feat = torch.nn.Parameter(torch.zeros(n, splatter.n_features, device=splatter.device))
        splatter.n_gaussians = g.pos.shape[0]
        if getattr(splatter, "use_filter3d", False):
            f3 = ckpt.get("filter3d")
            if f3 is not None and f3.numel() == n:
                splatter._set_filter3d(f3)
            else:
                splatter.compute_filter3d()
    if optimizer is not None and res is not None and res.get("optimizer") is not None:
        st = res["optimizer"]
        if st["kind"] == "torch":
            optimizer.load_state_dict(st["state"])
        else:
            optimizer.step_count = st["step"]
            for grp, lr in zip(optimizer.param_groups, st["lrs"]):
                grp["lr"] = lr
            optimizer._resume = (st["exp_avg"], st["exp_avg_sq"])      # consumed by FlatAdam._build
            if st.get("staged") is not None:
                optimizer._staged = st["staged"]
    bl = ckpt.get("bilagrid")
    if bilagrid is not None and bl is not None:
        if tuple(bl["grids"].shape) != tuple(bilagrid.grids.shape):
            raise ValueError(f"{path}: bilateral grids {list(bl['grids'].shape)} do not fit "
                             f"{list(bilagrid.grids.shape)}")
        with torch.no_grad():
            bilagrid.grids.copy_(bl["grids"])
        if bilagrid_optimizer is not None and bl.get("optimizer") is not None:
            bilagrid_optimizer.load_state_dict(bl["optimizer"])
    if restore_rng and res is not None:
        torch.set_rng_state(res["torch_rng"])
        if res.get("cuda_rng") is not None and splatter is not None:
            torch.cuda.set_rng_state(res["cuda_rng"], splatter.device)
        np.random.set_state(res["numpy_rng"])
    return ckpt
