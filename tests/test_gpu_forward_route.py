"""Inference propagation straight from the embedding tables.

`ops.propagate_mean_fused` takes E_0 as the pair (user table, item table): layer 1 gathers from the two tables and adds
them to the running sum where they are (`mmrec_spmm_steps_f32`'s two-block X / acc_in), the item-item product shares layer
1's launch, later layers are one ordinary launch each.  FREEDOM, BM3 and MGCN run it in inference; their outputs must be
the bits of the route it replaces: concatenate the tables, one SpMM launch per layer, then the item-item product with the
layer mean as its base.
"""
import ctypes

import numpy as np
import pytest
import torch

import bench
import test_gpu_exact_arith as X
from oracle import mmrec_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def _concat_route(A, ego, n_layers, post_csr=None, post_x=None, post_layers=1, post_row0=0, cooperative=True):
    """The route the models took before: torch.cat of the tables, one `spmm_raw` per layer with the running mean in its
    epilogue, then `mm_adj @ h` with the layer mean of the item rows as its base (freedom.py: `ops.spmm(mm_adj, h, base=i_g)`)."""
    from mmrec_b200 import ops
    e0 = torch.cat(ego) if isinstance(ego, (tuple, list)) else ego
    acc = torch.empty_like(e0)
    x = e0
    for l in range(1, n_layers + 1):
        last = l == n_layers
        y = None if last else torch.empty_like(e0)
        ops.spmm_raw(A, x, Y=y, acc_in=e0 if l == 1 else acc, acc_out=acc, acc_div=float(n_layers + 1) if last else 1.0)
        x = y
    if post_csr is not None:
        h = post_x
        for _ in range(post_layers - 1):
            y = torch.empty(post_csr.n_rows, h.shape[1], device=h.device)
            ops.spmm_raw(post_csr, h, Y=y)
            h = y
        out = torch.empty_like(acc[post_row0:])
        ops.spmm_raw(post_csr, h, acc_in=acc[post_row0:].contiguous(), acc_out=out)
        acc[post_row0:] = out
    return acc


@pytest.mark.parametrize("workload,model_name", [("tiny", "FREEDOM"), ("tiny", "BM3"), ("tiny", "MGCN"),
                                                 ("baby", "FREEDOM"), ("sports", "BM3"), ("clothing", "MGCN")])
def test_inference_forward_equals_concatenated_route(dev, monkeypatch, workload, model_name):
    from mmrec_b200 import ops
    wl = bench.Workload(workload, n_layers=3 if model_name == "FREEDOM" else 2)
    _, _, _, model = bench.build_model(wl, model_name, dev, {"n_ui_layers": wl.n_layers} if model_name == "FREEDOM" else None)
    model.eval()
    with torch.no_grad():
        bench.forward_eval(model)                                    # lazy inits (workspaces, occupancy queries)
        torch.cuda.synchronize()
        l0 = ops.launch_count()
        got = bench.forward_eval(model)
        n_launch = ops.launch_count() - l0
        calls = []
        monkeypatch.setattr(ops, "propagate_mean_fused", lambda *a, **k: calls.append(1) or _concat_route(*a, **k))
        want = bench.forward_eval(model)
    assert calls, "the model did not take the fused inference route"
    for g, w, what in zip(got, want, ("users", "items")):
        O.assert_bits(g, w, f"{model_name}/{workload} {what}")
    if model_name == "FREEDOM":
        assert n_launch <= model.n_ui_layers, n_launch              # was n_ui_layers + 1 SpMM launches (and a copy)


def _two_block(t, split, ld_hi):
    """(rows below `split`, rows from `split` on) of `t` in separate allocations; the second with leading dimension ld_hi."""
    lo = t[:split].clone()
    buf = torch.full((t.shape[0] - split, ld_hi), 9.0, device=t.device)
    buf[:, :t.shape[1]] = t[split:]
    return lo, buf[:, :t.shape[1]]


@pytest.mark.parametrize("cooperative", [0, 1])
@pytest.mark.parametrize("d", [32, 64, 256])
def test_steps_two_block_operands_bit_for_bit(dev, d, cooperative):
    """mmrec_spmm_steps_f32 with X and acc_in in two row blocks (own splits, the second block strided) against the exact
    result and against the same steps on the concatenated operands: a square matrix with split rows (513, 520, 4200
    non-zeros) and CTA-sized rows, splits that fall inside both, an independent product sharing the launch, the mean and
    `+ post` on the last rows."""
    from mmrec_b200 import _lib, ops
    from mmrec_b200.ops import CSR
    n, row, col, vals = X._spmm_matrix(11, n_fill=X.N_COLS - len(X.ROW_LENS))
    rng = np.random.default_rng(d + 5)
    Ai = X._csr_int(n, n, row, col, vals)
    E0 = O.exact_ints(rng, (n, d), 2)
    y = O.to_f32_exact(X._spmm_exact(Ai, E0), X.V_SCALE)
    n_post, row0 = 700, n - 700
    mr, mc = rng.integers(0, n_post, 5000), rng.integers(0, n_post, 5000)
    key = np.unique(mr * n_post + mc)
    mr, mc = key // n_post, key % n_post
    mv = O.exact_ints(rng, mr.shape, 2)
    mv[mv == 0] = 1
    xi = O.exact_ints(rng, (n_post, d), 2)
    h = O.to_f32_exact(X._spmm_exact(X._csr_int(n_post, n_post, mr, mc, mv), xi), X.V_SCALE)
    post = O.to_f32_exact(O.exact_ints(rng, (n_post, d), 5), 2.0 ** -4)
    _, want = O.spmm_epilogue_f32(y, O.to_f32_exact(E0, 1.0), 3.0)
    want[row0:] = (want[row0:] + post).astype(np.float32)

    A = CSR.from_coo(torch.from_numpy(row).to(dev), torch.from_numpy(col).to(dev), torch.from_numpy(O.to_f32_exact(vals, X.V_SCALE)).to(dev), n, n)
    M = CSR.from_coo(torch.from_numpy(mr).to(dev), torch.from_numpy(mc).to(dev), torch.from_numpy(O.to_f32_exact(mv, X.V_SCALE)).to(dev),
                     n_post, n_post)
    assert A.n_split == 3 and A.n_cta_tasks >= 1
    e0 = torch.from_numpy(O.to_f32_exact(E0, 1.0)).to(dev)
    x_post = torch.from_numpy(O.to_f32_exact(xi, 1.0)).to(dev)
    post_t = torch.from_numpy(post).to(dev)
    heavy = int(np.argmax(np.diff(Ai.indptr)))                       # the 4200-non-zero row
    lib = _lib.load()

    def run(Xop, Iop):
        Y, acc, hm = torch.empty(n, d, device=dev), torch.empty(n, d, device=dev), torch.empty(n_post, d, device=dev)
        steps = [ops._chain_step(A, Xop, Y=Y, acc_in=Iop, acc_out=acc, acc_div=3.0, post=post_t, post_row0=row0),
                 ops._chain_step(M, x_post, Y=hm)]
        arr = (_lib.SpmmStep2 * 2)(*steps)
        before = ops.launch_count()
        _lib.check(lib.mmrec_spmm_steps_f32(d, 2, ctypes.cast(arr, ctypes.c_void_p), cooperative, torch.cuda.current_stream().cuda_stream),
                   "mmrec_spmm_steps_f32")
        assert ops.launch_count() - before == 1
        return Y, acc, hm

    Yc, accc, hc = run(e0, e0)
    O.assert_bits(Yc, y, "concatenated Y")
    O.assert_bits(accc, want, "concatenated acc_out")
    O.assert_bits(hc, h, "independent product in the same launch")
    for xs, s_in in ((1000, 1000), (4, heavy), (n - 3, 1), (1, n - 1)):
        Y2, acc2, h2 = run(_two_block(e0, xs, d + 4), _two_block(e0, s_in, d + 8))
        O.assert_bits(Y2, Yc, f"two-block Y (x_split {xs}, acc_in_split {s_in})")
        O.assert_bits(acc2, accc, f"two-block acc_out (x_split {xs}, acc_in_split {s_in})")
        O.assert_bits(h2, hc, "independent product beside the two-block step")
    assert int(A.counters.abs().sum().item()) == 0 and int(M.counters.abs().sum().item()) == 0


def test_propagate_mean_fused_two_tables_equals_tensor(dev):
    """The pair form with post, ordinary launches, against the tensor form (one cooperative launch), several layers."""
    from mmrec_b200 import ops
    from mmrec_b200.ops import CSR
    gen = torch.Generator().manual_seed(4)
    U, I, d = 900, 500, 64
    r = torch.randint(0, U, (7000,), generator=gen); c = torch.randint(0, I, (7000,), generator=gen)
    r = torch.cat([r, torch.full((1500,), 3)]); c = torch.cat([c, torch.randint(0, I, (1500,), generator=gen)])
    v = torch.rand(r.numel(), generator=gen) - 0.5
    A = CSR.from_coo(torch.cat([r, c + U]).to(dev), torch.cat([c + U, r]).to(dev), torch.cat([v, v]).to(dev), U + I, U + I, symmetric=True)
    M = CSR.from_coo(torch.randint(0, I, (4000,), generator=gen).to(dev), torch.randint(0, I, (4000,), generator=gen).to(dev),
                     torch.rand(4000, generator=gen).to(dev), I, I)
    ue, ie = torch.randn(U, d, generator=gen).to(dev), torch.randn(I, d, generator=gen).to(dev)
    for L, P in ((3, 1), (1, 1), (2, 2), (3, 0)):
        kw = dict(post_csr=M, post_x=ie, post_layers=P, post_row0=U) if P else {}
        want = ops.propagate_mean_fused(A, torch.cat([ue, ie]), L, **kw)
        before = ops.launch_count()
        got = ops.propagate_mean_fused(A, (ue, ie), L, cooperative=False, **kw)
        assert ops.launch_count() - before == (max(L - 1, P) + 1 if P else L), (L, P)   # the last layer waits for h
        O.assert_bits(got, want, f"L={L} post_layers={P}")
        O.assert_bits(got, _concat_route(A, (ue, ie), L, M if P else None, ie, max(P, 1), U), f"L={L} post_layers={P} vs concatenated")
