"""The visible-only Adam oracle (tests/visible_adam_oracle.py) against torch.optim.Adam, and the union of the
visibility masks over 2 gloo ranks (dp.all_reduce_visible).  CPU only."""
import os
import socket
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import visible_adam_oracle as VO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-gaussian-splatting_b200"))

WIDTHS = (3, 27, 1, 4, 3)            # pos, rgb (SH degree 2), opa, quat, scale
LRS = (0.003, 0.03, 0.05, 0.004, 0.005)
BETAS, EPS = (0.9, 0.99), 1e-8


def _buffers(n, seed):
    gen = torch.Generator().manual_seed(seed)
    starts, total = VO.layout(n, WIDTHS)
    p = torch.randn(total, generator=gen)
    return starts, total, p, torch.zeros(total), torch.zeros(total), gen


def test_oracle_equals_torch_adam_on_the_gathered_rows():
    """The equivalence, spelled out.  At global step t the visible rows get the update a torch.optim.Adam would give
    a parameter made of exactly those rows, p[vis], whose state is their own moments (m[vis], v[vis]) and whose step
    counter stands at t - 1: the rows with a zero gradient are removed from the parameter instead of being stepped,
    and because torch's counter is forced to the global one each iteration, the bias corrections 1 - beta^t are the
    global step's however rarely a row was seen.  The mask changes every iteration."""
    n = 203
    starts, total, p, m, v, gen = _buffers(n, 0)
    ref_p, ref_m, ref_v = p.clone(), m.clone(), v.clone()
    before_pad = [(s0 + n * w, p[s0 + n * w:(s0 + n * w + 3) // 4 * 4].clone()) for s0, w in zip(starts, WIDTHS)]
    for t in range(1, 8):
        vis = (torch.rand(n, generator=gen) < 0.4).to(torch.uint8)
        g = torch.randn(total, generator=gen) * (0.1 * t)
        rows = vis.bool()
        for s0, w, lr in zip(starts, WIDTHS, LRS):
            sl = slice(s0, s0 + n * w)
            q = torch.nn.Parameter(ref_p[sl].view(n, w)[rows].clone())
            opt = torch.optim.Adam([q], lr=lr, betas=BETAS, eps=EPS)
            opt.state[q] = dict(step=torch.tensor(float(t - 1)), exp_avg=ref_m[sl].view(n, w)[rows].clone(),
                                exp_avg_sq=ref_v[sl].view(n, w)[rows].clone())
            q.grad = g[sl].view(n, w)[rows].clone()
            opt.step()
            ref_p[sl].view(n, w)[rows] = q.detach()
            ref_m[sl].view(n, w)[rows] = opt.state[q]["exp_avg"]
            ref_v[sl].view(n, w)[rows] = opt.state[q]["exp_avg_sq"]
        VO.adam_visible(p, g, m, v, starts, WIDTHS, LRS, n, vis, *BETAS, EPS, t)
    for got, want in ((p, ref_p), (m, ref_m), (v, ref_v)):
        assert float((got - want).abs().max()) <= 2e-6 * float(want.abs().max())
    for o, pad in before_pad:
        assert torch.equal(p[o:o + pad.numel()], pad)          # pads are nobody's row


def test_oracle_all_visible_is_dense_adam_and_none_visible_is_identity():
    n = 64
    starts, total, p, m, v, gen = _buffers(n, 1)
    q = torch.nn.Parameter(p.clone())
    g = torch.randn(total, generator=gen)
    frozen = [t.clone() for t in (p, m, v)]
    VO.adam_visible(p, g, m, v, starts, WIDTHS, LRS, n, torch.zeros(n, dtype=torch.uint8), *BETAS, EPS, 1)
    assert all(torch.equal(a, b) for a, b in zip((p, m, v), frozen))
    one_lr = (0.01,) * len(WIDTHS)
    opt = torch.optim.Adam([q], lr=0.01, betas=BETAS, eps=EPS)
    for t in range(1, 4):
        q.grad = g * t
        opt.step()
        VO.adam_visible(p, g * t, m, v, starts, WIDTHS, one_lr, n, torch.ones(n, dtype=torch.uint8), *BETAS, EPS, t)
    for s0, w in zip(starts, WIDTHS):
        sl = slice(s0, s0 + n * w)
        assert float((p[sl] - q.detach()[sl]).abs().max()) <= 2e-6 * float(q.detach().abs().max())


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import dp
    mask = torch.tensor([1, 0, 0, 1, 0, 0, 1, 0] if rank == 0 else [0, 0, 1, 1, 0, 1, 0, 0], dtype=torch.uint8)
    ret = dp.all_reduce_visible(mask)
    out[rank] = (mask.tolist(), ret.data_ptr() == mask.data_ptr(), str(mask.dtype))
    dist.destroy_process_group()


def test_all_reduce_visible_is_the_union_world2():
    world, port = 2, _free_port()
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
    for r in range(world):
        assert out[r] == ([1, 0, 1, 1, 0, 1, 1, 0], True, "torch.uint8")


def test_all_reduce_visible_without_a_group_is_the_identity():
    import dp
    mask = torch.tensor([1, 0, 1], dtype=torch.uint8)
    assert dp.all_reduce_visible(mask) is mask and mask.tolist() == [1, 0, 1]
