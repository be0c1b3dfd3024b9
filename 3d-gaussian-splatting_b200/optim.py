"""Fused flat-bucket Adam (SURVEY.md §8 f-2).

Drop-in for the way the reference steps its optimizer (train.py:56-64 / :173-181:
`torch.optim.Adam([{"params": p, "lr": lr} x 5], betas=(0.9, 0.99))`, learning rates rewritten in
`param_groups[i]["lr"]` every iteration, train.py:184-185): same constructor shape, `zero_grad`,
`step`, `param_groups`.  The fused backward leaves the five gradients as views of ONE flat buffer
(renderer._flat_grads; all-reduced in place by dp.GradBucket), so the step is a single kernel
(`gaussian.adam_step` -> `gs_adam_step`) over flat parameter / moment buffers instead of
5 x (foreach) kernel groups.  No CPU / torch fallback: gradients that are not one flat bucket are
an error.

`step(visible=mask)` is a second optimizer, opt-in: Adam on the rows of the Gaussians the last frames binned
(`Splatter.visible_mask()`), the "sparse Adam" of 3DGS / gsplat's `SelectiveAdam`
(`gaussian.adam_step_visible` -> `gs_adam_step_visible`).  A Gaussian that was not seen is frozen, moments included,
where dense Adam lets it drift on its momentum; the bias corrections use the global step count either way.
"""
from __future__ import annotations

from typing import List

import torch

import gaussian


class FlatAdam:
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.99), eps=1e-8):
        groups = list(params)
        if groups and not isinstance(groups[0], dict):
            groups = [{"params": groups}]
        self.param_groups: List[dict] = []
        for g in groups:
            ps = g["params"]
            ps = [ps] if isinstance(ps, torch.Tensor) else list(ps)
            self.param_groups.append({"params": ps, "lr": float(g.get("lr", lr))})
        self.betas, self.eps = (float(betas[0]), float(betas[1])), float(eps)
        self.step_count = 0
        self._flat = None          # (flat_param, exp_avg, exp_avg_sq, ordered params, segment ends)
        self._staged = None        # moments carried over a change of n: see replace_params
        self._zero_rows = None     # rows whose restored moments the next _build zeroes: see zero_moment_rows

    def zero_grad(self, set_to_none: bool = True):
        for g in self.param_groups:
            for p in g["params"]:
                if set_to_none:
                    p.grad = None
                elif p.grad is not None:
                    p.grad.zero_()

    def _lr_of(self, p):
        for g in self.param_groups:
            if any(p is q for q in g["params"]):
                return g["lr"]
        raise KeyError("parameter not in any group")

    def _build(self, ordered):
        """Move the parameters into one flat buffer laid out exactly like the gradient bucket."""
        g0 = ordered[0].grad
        base = g0.storage_offset()
        span_end = ordered[-1].grad.storage_offset() + ordered[-1].grad.numel()
        total = (span_end - base + 3) // 4 * 4
        dev = g0.device
        flat = torch.zeros(total, device=dev, dtype=torch.float32)
        ends = []
        for i, p in enumerate(ordered):
            o = p.grad.storage_offset() - base
            view = flat[o:o + p.numel()].view(p.shape)
            view.copy_(p.data)
            p.data = view                                   # the Parameter now aliases the flat buffer
            nxt = ordered[i + 1].grad.storage_offset() - base if i + 1 < len(ordered) else total
            ends.append(nxt)
        m, v = torch.zeros_like(flat), torch.zeros_like(flat)
        resume = getattr(self, "_resume", None)          # moments restored by checkpoint.load_checkpoint
        if resume is not None and resume[0] is not None and resume[0].numel() == flat.numel():
            m.copy_(resume[0])
            v.copy_(resume[1])
            self._keep_step = True
        self._resume = None
        if self._staged is not None:                     # the old rows lead each segment; the new rows stay zero
            everyone = self._all_params()
            for p in ordered:
                k = next(i for i, q in enumerate(everyone) if q is p)
                if self._staged[k] is not None:
                    o, sm, sv = p.data.storage_offset(), self._staged[k][0], self._staged[k][1]
                    m[o:o + sm.numel()].copy_(sm.reshape(-1))
                    v[o:o + sv.numel()].copy_(sv.reshape(-1))
            self._staged = None
            self._keep_step = True
        if self._zero_rows is not None:                  # rows relocated between a checkpoint load and this build
            rows = self._zero_rows.to(flat.device)
            for p in ordered:
                if p.dim() and p.shape[0] == rows.numel():
                    o = p.data.storage_offset()
                    for t in (m, v):
                        t[o:o + p.numel()].view(rows.numel(), -1).masked_fill_(rows.view(-1, 1), 0.0)
            self._zero_rows = None
        self._flat = (flat, m, v, ordered, ends, base)

    def _all_params(self):
        return [p for g in self.param_groups for p in g["params"]]

    def live_moments(self, params):
        """(exp_avg, exp_avg_sq, starts, widths) of the flat moment buffers when every parameter they hold is one of
        `params` and still aliases the flat buffer (all with the same row count), else None (before the first step,
        or after `replace_params` until the next one)."""
        if self._flat is None or self._staged is not None:
            return None
        flat, m, v, ordered, _, _ = self._flat
        store = flat.untyped_storage().data_ptr()
        if any(not any(p is q for q in params) for p in ordered) \
                or any(p.data.untyped_storage().data_ptr() != store for p in ordered):
            return None
        n = ordered[0].shape[0]
        return m, v, [p.data.storage_offset() for p in ordered], [p.numel() // max(n, 1) for p in ordered]

    @torch.no_grad()
    def zero_moment_rows(self, rows):
        """Zero the moments of rows `rows` (bool [n]) of every parameter with n rows while they are not in a live
        flat buffer (`live_moments` is None): the moments `replace_params` staged, and the moments a checkpoint
        restored, which the next `_build` places and then zeroes at those rows.  Exact zeros; nothing else changes."""
        for s in self._staged or []:
            for t in s or ():
                if t.dim() and t.shape[0] == rows.numel():
                    t.masked_fill_(rows.to(t.device).view((-1,) + (1,) * (t.dim() - 1)), 0.0)
        resume = getattr(self, "_resume", None)
        if resume is not None and resume[0] is not None:
            self._zero_rows = rows.clone() if self._zero_rows is None else self._zero_rows | rows

    @torch.no_grad()
    def replace_params(self, pairs):
        """Point `param_groups` at new Parameters, `pairs` = [(old, new)], where the first rows of each new Parameter
        continue the old one's rows (growth).  The moments of the old rows are staged and the next step's `_build`
        puts them in the first rows of the new segments and zeroes the rest; `step_count` is kept.  A checkpoint taken
        before that step saves the staged moments."""
        old = self._all_params()
        staged = list(self._staged) if self._staged is not None else [None] * len(old)
        if self._staged is None and self._flat is not None:
            flat, m, v, ordered, _, _ = self._flat
            store = flat.untyped_storage().data_ptr()
            for k, p in enumerate(old):
                if any(p is q for q in ordered) and p.data.untyped_storage().data_ptr() == store:
                    o = p.data.storage_offset()
                    staged[k] = (m[o:o + p.numel()].view(p.shape), v[o:o + p.numel()].view(p.shape))
        for g in self.param_groups:
            g["params"] = [next((nw for od, nw in pairs if od is p), p) for p in g["params"]]
        self._staged = staged if any(s is not None for s in staged) else None
        self._flat = None

    @torch.no_grad()
    def step(self, visible=None):
        """One Adam step.  `visible` None: every float of the bucket (dense).  A CUDA uint8 tensor [n]: only the rows
        i with visible[i] != 0 of every parameter (each must have shape[0] == n); the others keep their value and
        their moments, bit for bit.  `step_count` advances by one either way."""
        params = [p for g in self.param_groups for p in g["params"] if p.grad is not None]
        if not params:
            return
        ordered = sorted(params, key=lambda p: p.grad.storage_offset())
        g0 = ordered[0].grad
        store = g0.untyped_storage().data_ptr()
        for a, b in zip(ordered[:-1], ordered[1:]):
            gap = b.grad.storage_offset() - (a.grad.storage_offset() + a.grad.numel())
            if b.grad.untyped_storage().data_ptr() != store or not (0 <= gap <= 3):
                raise RuntimeError("FlatAdam needs the gradients to be views of one flat bucket "
                                   "(as produced by renderer.render_frame / render_frame_final)")
        if self._flat is None or len(self._flat[3]) != len(ordered) or any(a is not b for a, b in zip(self._flat[3], ordered)) \
                or any(p.data.untyped_storage().data_ptr() != self._flat[0].untyped_storage().data_ptr() for p in ordered):
            self._build(ordered)
            if not getattr(self, "_keep_step", False):
                self.step_count = 0
            self._keep_step = False
        flat, m, v, _, ends, _ = self._flat
        base = g0.storage_offset()
        gflat = torch.empty(0, dtype=torch.float32, device=g0.device).set_(g0.untyped_storage(), base, (flat.numel(),))
        if (base * 4 + g0.untyped_storage().data_ptr()) % 16:
            raise RuntimeError("FlatAdam: gradient bucket must be 16-byte aligned")
        lrs = [self._lr_of(p) for p in ordered]
        if visible is None:
            self.step_count += 1
            gaussian.adam_step(flat, gflat, m, v, ends, lrs, self.betas[0], self.betas[1], self.eps, self.step_count)
            return
        if not (torch.is_tensor(visible) and visible.is_cuda and visible.dtype == torch.uint8 and visible.dim() == 1):
            raise TypeError("FlatAdam.step: visible must be a 1-D CUDA uint8 tensor (Splatter.visible_mask())")
        n = visible.numel()
        if any(p.dim() == 0 or p.shape[0] != n for p in ordered):
            raise ValueError(f"FlatAdam.step: visible has {n} entries but the parameters have "
                             f"{[tuple(p.shape) for p in ordered]}: every parameter needs shape[0] == visible.numel()")
        starts = [p.grad.storage_offset() - base for p in ordered]
        widths = [p.numel() // n if n else 1 for p in ordered]
        self.step_count += 1
        gaussian.adam_step_visible(flat, gflat, m, v, starts, widths, lrs, visible.contiguous(), self.betas[0],
                                   self.betas[1], self.eps, self.step_count)
