"""f1 (csrc/train.cu, mmrec_b200/optim.py): projection backward and the Adam step against torch's own fp32 / fp64 arithmetic.

Reference behaviour: autograd of `nn.Linear` over the trainable modality tables (src/models/freedom.py:58-62,205-209) and
`optim.Adam(...).step()` (src/common/trainer.py:117-118,189).  Floating point: 2e-6 relative (Frobenius) against fp64
products; after three optimiser steps on the same gradients, parameters within 2e-6 and moments within 5e-6 of
torch.optim.Adam (FusedAdam on a model: 1e-5 / 1e-4).  These are norms over whole tensors; tests/test_gpu_exact_arith.py
compares the same kernels bit for bit.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 2e-6


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize("n_idx,n_rows,d", [(0, 10, 64), (1, 1, 1), (4096, 7000, 64), (20000, 300, 100), (9000, 70, 256), (500, 100000, 32),
                                            (700, 333, 300)])
def test_index_sum_rows(dev, n_idx, n_rows, d):
    from mmrec_b200 import ops
    g = torch.Generator().manual_seed(n_idx + d)
    idx = torch.randint(0, n_rows, (n_idx,), generator=g)
    x = torch.randn(n_idx, d, generator=g)
    want = torch.zeros(n_rows, d, dtype=torch.float64).index_add_(0, idx, x.double())
    got = ops.index_sum_rows(x.to(dev), idx.to(dev), n_rows)
    assert got.shape == (n_rows, d)
    assert rel(got, want) < TOL if n_idx else float(got.abs().max()) == 0.0
    again = ops.index_sum_rows(x.to(dev), idx.to(dev), n_rows)
    assert torch.equal(got, again)                                   # ascending-j sums: bit-reproducible


@pytest.mark.parametrize("n,n_table,F,d,gather,bias", [
    (7000, 7000, 4096, 64, False, True),          # BM3 / MGCN: the whole image table
    (4096, 7000, 4096, 64, True, True),           # FREEDOM: pos + neg items of a 2048-sample batch
    (7000, 7000, 384, 64, False, True),           # text table (one column strip, partly empty)
    (1000, 1000, 516, 128, False, False),         # d = 128: two k tiles; F not a multiple of the strip
    (37, 50, 100, 20, True, True),                # small and ragged
    (333, 333, 130, 64, False, True),             # F not a multiple of 4: 4-byte accesses
    (50, 64, 77, 300, True, True),
    (1, 1, 4, 1, False, True),
])
def test_linear_wgrad(dev, n, n_table, F, d, gather, bias):
    from mmrec_b200 import ops
    g = torch.Generator().manual_seed(n + F + d)
    table = torch.randn(n_table, F, generator=g)
    up = torch.randn(n, d, generator=g)
    idx = torch.randint(0, n_table, (n,), generator=g) if gather else None
    x = table if idx is None else table[idx]
    want_w = up.double().t().mm(x.double())
    want_b = up.double().sum(0)
    dW, db = ops.linear_wgrad(up.to(dev), table.to(dev), None if idx is None else idx.to(dev), want_bias=bias)
    assert dW.shape == (d, F) and rel(dW, want_w) < TOL
    if bias:
        assert rel(db, want_b) < TOL
    else:
        assert db is None
    dW2, _ = ops.linear_wgrad(up.to(dev), table.to(dev), None if idx is None else idx.to(dev), want_bias=bias)
    assert torch.equal(dW, dW2)                                      # fixed reduction order


def test_linear_wgrad_empty(dev):
    from mmrec_b200 import ops
    dW, db = ops.linear_wgrad(torch.zeros(0, 8, device=dev), torch.randn(5, 16, device=dev))
    assert float(dW.abs().max()) == 0.0 and float(db.abs().max()) == 0.0


@pytest.mark.parametrize("n_rows,F,d", [(7000, 4096, 64), (7000, 384, 64), (333, 1028, 128), (17, 8, 3), (1, 4, 1), (5000, 512, 96),
                                        (333, 130, 64), (129, 200, 256), (50, 77, 300)])
def test_linear_dgrad(dev, n_rows, F, d):
    from mmrec_b200 import ops
    g = torch.Generator().manual_seed(n_rows + F + d)
    G = torch.randn(n_rows, d, generator=g)
    W = torch.randn(d, F, generator=g)
    got = ops.linear_dgrad(G.to(dev), W.to(dev))
    assert got.shape == (n_rows, F) and rel(got, G.double().mm(W.double())) < TOL


def _torch_adam_reference(p0, grads, lr, wd, betas=(0.9, 0.999), eps=1e-8):
    p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([p], lr=lr, weight_decay=wd, betas=betas, eps=eps)
    for g in grads:
        p.grad = g.clone()
        opt.step()
    st = opt.state[p]
    return p.detach(), st["exp_avg"], st["exp_avg_sq"]


@pytest.mark.parametrize("n_rows,F,d,wd", [(7000, 4096, 64, 0.0), (1500, 384, 64, 0.01), (300, 260, 128, 0.0), (9, 4, 5, 0.1)])
def test_linear_dgrad_adam_matches_torch_adam(dev, n_rows, F, d, wd):
    """Three Adam steps of a table whose gradient is G @ W, fused, against torch.optim.Adam on the materialised gradient."""
    from mmrec_b200 import ops
    gen = torch.Generator().manual_seed(n_rows + F)
    p0 = torch.randn(n_rows, F, generator=gen).to(dev)
    W = (0.1 * torch.randn(d, F, generator=gen)).to(dev)
    Gs = [(0.05 * torch.randn(n_rows, d, generator=gen)).to(dev) for _ in range(3)]
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    want_p, want_m, want_v = _torch_adam_reference(p0, [g.double().mm(W.double()).float() for g in Gs], lr, wd)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for t, G in enumerate(Gs, 1):
        ops.linear_dgrad_adam(G, W, p, m, v, b1, b2, eps, wd, -lr / (1 - b1 ** t), (1 - b2 ** t) ** 0.5)
    assert rel(m, want_m) < 5e-6 and rel(v, want_v) < 5e-6
    assert rel(p - p0, want_p - p0) < 1e-4         # the update itself: 3 steps of ~lr on values ~1 (fp32 spacing of p: ~2e-5 of it)
    assert rel(p, want_p) < TOL


def test_adam_step_matches_torch_adam(dev):
    from mmrec_b200 import ops
    gen = torch.Generator().manual_seed(5)
    shapes = [(20000, 64), (7000, 64), (64, 4096), (64,), (1,), (4097,), (3, 5, 7)] + [(11,)] * 30    # > 24 tensors: two launches
    ps = [torch.randn(*s, generator=gen).to(dev) for s in shapes]
    steps = [[(0.1 * torch.randn(*s, generator=gen)).to(dev) for s in shapes] for _ in range(3)]
    lr, wd, b1, b2, eps = 2e-3, 0.05, 0.9, 0.999, 1e-8
    want = [_torch_adam_reference(p, [st[i] for st in steps], lr, wd) for i, p in enumerate(ps)]
    cur = [p.clone() for p in ps]
    ms, vs = [torch.zeros_like(p) for p in ps], [torch.zeros_like(p) for p in ps]
    # an unaligned view: element 1.. of a buffer (scalar path of the kernel)
    buf = torch.zeros(4097 + 1, device=dev)
    cur[5] = buf[1:]; cur[5].copy_(ps[5])
    for t, grads in enumerate(steps, 1):
        ops.adam_step([(cur[i], grads[i], ms[i], vs[i], -lr / (1 - b1 ** t), (1 - b2 ** t) ** 0.5) for i in range(len(ps))], b1, b2, eps, wd)
    for i in range(len(ps)):
        assert rel(cur[i], want[i][0]) < TOL, shapes[i]
        assert rel(ms[i], want[i][1]) < 5e-6 and rel(vs[i], want[i][2]) < 5e-6


@pytest.mark.parametrize("gather", [False, True])
def test_project_backward_matches_autograd(dev, gather):
    """`ops.project` under autograd (wgrad / index_sum_rows / dgrad kernels) against torch's own backward of the same expression."""
    from mmrec_b200 import ops
    gen = torch.Generator().manual_seed(3)
    table = torch.randn(900, 256, generator=gen).to(dev).requires_grad_()
    lin = torch.nn.Linear(256, 64).to(dev)
    idx = torch.randint(0, 900, (1300,), generator=gen).to(dev) if gather else None
    up = torch.randn(1300 if gather else 900, 64, generator=gen).to(dev)
    y = ops.project(table, lin.weight, lin.bias, idx=idx)
    (y * up).sum().backward()
    got = table.grad.clone(), lin.weight.grad.clone(), lin.bias.grad.clone()
    table.grad = None; lin.zero_grad()
    t64, w64, b64 = table.detach().double().requires_grad_(), lin.weight.detach().double().requires_grad_(), lin.bias.detach().double().requires_grad_()
    y2 = torch.nn.functional.linear(t64, w64, b64)
    y2 = y2 if idx is None else y2[idx]
    (y2 * up.double()).sum().backward()
    for g, w in zip(got, (t64.grad, w64.grad, b64.grad)):
        assert rel(g, w) < TOL


@pytest.mark.parametrize("gather,accumulate,factored", [(False, False, True), (True, False, True), (True, True, True), (True, False, False)])
def test_fused_adam_equals_torch_adam_on_a_projection_model(dev, gather, accumulate, factored):
    """FusedAdam (factored table gradient, never materialised) against torch.optim.Adam on the same tiny model: parameters and
    optimiser state after 4 steps.  `accumulate`: two backwards per step -- the factored form must fall back to the dense one."""
    from mmrec_b200 import ops
    from mmrec_b200.optim import FusedAdam

    def make():
        gen = torch.Generator().manual_seed(11)
        table = torch.nn.Parameter(torch.randn(500, 128, generator=gen).to(dev))
        lin = torch.nn.Linear(128, 64).to(dev)
        with torch.no_grad():
            lin.weight.copy_(0.1 * torch.randn(64, 128, generator=gen)); lin.bias.copy_(0.1 * torch.randn(64, generator=gen))
        emb = torch.nn.Parameter(torch.randn(500, 64, generator=gen).to(dev))
        return table, lin, emb

    def loss_fn(table, lin, emb, idx, ours):
        proj = ops.project(table, lin.weight, lin.bias, idx=idx) if ours else \
            (torch.nn.functional.linear(table, lin.weight, lin.bias) if idx is None else torch.nn.functional.linear(table, lin.weight, lin.bias)[idx])
        e = emb if idx is None else emb[idx]
        return (proj * e).sum(1).sigmoid().log().neg().mean()

    gen = torch.Generator().manual_seed(12)
    idxs = [torch.randint(0, 500, (700,), generator=gen).to(dev) if gather else None for _ in range(8)]
    a, b = make(), make()
    opt_a = FusedAdam([a[0], *a[1].parameters(), a[2]], lr=1e-2, weight_decay=0.0, factored=factored)
    opt_b = torch.optim.Adam([b[0], *b[1].parameters(), b[2]], lr=1e-2, weight_decay=0.0)
    for s in range(4):
        opt_a.zero_grad(); opt_b.zero_grad()
        for r in range(2 if accumulate else 1):
            loss_fn(*a, idxs[2 * s + r], True).backward()
            loss_fn(*b, idxs[2 * s + r], False).backward()
        if factored and not accumulate:
            assert a[0].grad is None and a[0]._mmrec_pending is not None       # the dense table gradient was never built
        if not factored:
            assert a[0].grad is not None and a[0]._mmrec_pending is None
        v0 = a[0]._version
        opt_a.step(); opt_b.step()
        assert a[0]._version > v0 and a[0]._mmrec_pending is None
    pa = [a[0], *a[1].parameters(), a[2]]
    pb = [b[0], *b[1].parameters(), b[2]]
    for x, y in zip(pa, pb):
        assert rel(x, y) < 1e-5
        assert rel(opt_a.state[x]["exp_avg"], opt_b.state[y]["exp_avg"]) < 1e-4
        assert float(opt_a.state[x]["step"]) == float(opt_b.state[y]["step"]) == 4.0
    # state_dict layout is torch.optim.Adam's
    sd = opt_a.state_dict()
    assert set(sd["state"][0]) == {"step", "exp_avg", "exp_avg_sq"} and sd["param_groups"][0]["lr"] == 1e-2
