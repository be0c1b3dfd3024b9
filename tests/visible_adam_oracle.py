"""Visible-only Adam (gs_adam_step_visible) restated in fp32 torch over the segment layout of the flat bucket.

Segment s is the row-major [n_rows, widths[s]] array at float starts[s] of the flat buffers (each start a multiple of
4, as renderer._flat_grads lays the gradients out).  Row i of every segment is updated when visible[i] != 0; every
other float, pads included, is left alone.  The bias corrections come from the global step, not from how often a row
was seen."""
import math

import torch


def layout(n_rows, widths):
    """(starts, total): segments in order, each padded to a multiple of 4 floats."""
    starts, o = [], 0
    for w in widths:
        starts.append(o)
        o += (n_rows * w + 3) // 4 * 4
    return starts, o


def adam_visible(p, g, m, v, starts, widths, lrs, n_rows, visible, beta1, beta2, eps, step):
    """In place on the flat fp32 CPU tensors p, m, v."""
    rows = visible.bool()
    f32 = torch.float32
    b1, b2 = torch.tensor(beta1, dtype=f32), torch.tensor(beta2, dtype=f32)
    bc1 = 1.0 - float(b1) ** step
    bc2 = 1.0 - float(b2) ** step
    inv = torch.tensor(1.0 / math.sqrt(bc2), dtype=f32)
    for s0, w, lr in zip(starts, widths, lrs):
        sl = slice(s0, s0 + n_rows * w)
        pv, gv, mv, vv = (t[sl].view(n_rows, w) for t in (p, g, m, v))
        gg, mm, v2 = gv[rows], mv[rows], vv[rows]
        mm = mm + (1 - b1) * (gg - mm)
        v2 = b2 * v2 + (1 - b2) * gg * gg
        step_size = torch.tensor(float(torch.tensor(lr, dtype=f32)) / bc1, dtype=f32)
        pv[rows] = pv[rows] - step_size * (mm / (v2.sqrt() * inv + torch.tensor(eps, dtype=f32)))
        mv[rows] = mm
        vv[rows] = v2
