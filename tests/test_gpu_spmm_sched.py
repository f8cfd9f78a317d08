"""K1 SpMM (csrc/spmm.cu): the summation order, restated on the host and pinned bit for bit on general fp32 data.

The exact-arithmetic tests (test_gpu_exact_arith.py, test_gpu_spmm_scale.py) use operands whose partial sums are exact, so
they pass under any order of the adds.  Who runs a task -- a lane group, a warp, a whole CTA -- is free; the order of its
arithmetic is not, and only inexact data can see it.  The order, for a work plan (`mmrec_spmm_plan`) and T lanes per task:

* a task of at most light_max non-zeros: one fmaf chain over its entries, from +0;
* a longer task: G = 256 / T chunks of ceil(len / G) consecutive entries, each an fmaf chain from +0, the chunk sums added
  in chunk order from +0, whoever runs it;
* a split row: the sums of its segments added in segment order, from +0;
* without the plan: one fmaf chain per row.

`restate` computes this in numpy with `oracle.fmaf32` (CUDA's fmaf, rounded once) and fp32 adds; the device must match it
at every lane instance, at the widths 3d, with and without the plan and under the edge-keep mask.  The graph has light
rows, rows of the CTA list from light_max + 1 to a whole segment and at multiples of every G, split rows, and more tasks
than the grid has warps (asserted).  Columns are independent, so one restatement at width 384 serves every width d <= 384 that has
the same G.
"""
import numpy as np
import pytest
import torch

from oracle import mmrec_oracle as O
from test_gpu_spmm_scale import _Lanes, _default_lanes, _lane_instances, _sms, plan_np

pytestmark = pytest.mark.gpu

MID = 256                      # CTA-list tasks on both sides of this length: one load batch per lane group, or several
DMAX = 384
ACC_DIV = 3.0


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


class _Sched:
    """A 12k x 8k matrix with random fp32 values: rows of 0-32 non-zeros, rows of the CTA list at and around light_max + 1,
    the multiples of G = 8 ... 128 and the segment length, and split rows up to 5,000 non-zeros; X and acc_in N(0, 1) fp32."""

    def __init__(self, dev):
        from mmrec_b200 import ops
        rng = np.random.default_rng(11)
        n_rows, n_cols = 12000, 8000
        marks = [33, 34, 63, 64, 65, 127, 128, 129, 200, 255, 256, 257, 258, 300, 384, 511, 512]
        lens = np.concatenate([rng.integers(0, 33, n_rows - 560 - 6), np.repeat(marks, 10), rng.integers(33, 513, 390),
                               [513, 700, 1024, 1025, 3000, 5000]])
        rng.shuffle(lens)
        rows = np.repeat(np.arange(n_rows), lens)
        cols = np.concatenate([np.sort(rng.choice(n_cols, n, replace=False)) for n in lens])
        vals = rng.standard_normal(rows.size).astype(np.float32)
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
        self.A = ops.CSR.from_coo(t(rows, torch.int64), t(cols, torch.int64), t(vals, torch.float32), n_rows, n_cols,
                                  sum_duplicates=False)
        self.rowptr = self.A.rowptr.cpu().numpy().astype(np.int64)
        self.colidx = self.A.colidx[:self.A.nnz].cpu().numpy().astype(np.int64)
        self.vals = self.A.vals[:self.A.nnz].cpu().numpy()
        self.X = rng.standard_normal((n_cols, DMAX)).astype(np.float32)
        self.acc_in = rng.standard_normal((n_rows, DMAX)).astype(np.float32)
        self.plan = plan_np(self.rowptr, self.A.seg, self.A.light_max)
        self.n_rows, self.n_cols = n_rows, n_cols
        self._ref = {}

    def restate(self, G, use_plan=True, keep=None, scale=1.0):
        """Y = A X in the kernel's order for G chunks per CTA-list task (width DMAX)."""
        key = (G, use_plan, keep is not None)
        if key in self._ref:
            return self._ref[key]
        w = self.vals if keep is None else np.where(keep, (self.vals * np.float32(scale)).astype(np.float32), np.float32(0))
        if not use_plan:
            out = _chains(self.rowptr[:-1], np.diff(self.rowptr), w, self.colidx, self.X, keep)
            self._ref[key] = out
            return out
        tk = self.plan["tasks"].astype(np.int64)
        b, e = tk[:, 1], tk[:, 2]
        n = e - b
        cta = n > self.A.light_max
        # chains: one per light task, G per CTA-list task (chunk k: [b + k c, min(e, b + (k + 1) c)), possibly empty)
        c = -(-n[cta] // G)
        kb = b[cta][:, None] + np.arange(G)[None, :] * c[:, None]
        kl = np.clip(e[cta][:, None] - kb, 0, c[:, None])
        starts = np.concatenate([b[~cta], kb.ravel()])
        lens = np.concatenate([n[~cta], kl.ravel()])
        ch = _chains(starts, lens, w, self.colidx, self.X, keep)
        task_sum = np.empty((tk.shape[0], DMAX), np.float32)
        n_light = int((~cta).sum())
        task_sum[~cta] = ch[:n_light]
        chunks = ch[n_light:].reshape(-1, G, DMAX)
        s = np.zeros((chunks.shape[0], DMAX), np.float32)
        for k in range(G):                                       # chunk order, from +0
            s = s + chunks[:, k]
        task_sum[cta] = s
        out = np.zeros((self.n_rows, DMAX), np.float32)
        whole = tk[:, 3] < 0
        out[tk[whole, 0]] = task_sum[whole]
        seg = self.A.seg
        for sid, (_, n_seg, rb, _) in enumerate(self.plan["split_rows"].astype(np.int64)):
            idx = np.nonzero(tk[:, 3] == sid)[0]
            idx = idx[np.argsort((tk[idx, 1] - rb) // seg)]
            assert idx.size == n_seg
            acc = np.zeros(DMAX, np.float32)
            for t in idx:                                        # segment order, from +0
                acc = acc + task_sum[t]
            out[tk[idx[0], 0]] = acc
        self._ref[key] = out
        return out


def _chains(starts, lens, w, colidx, X, keep=None):
    """fmaf chains from +0 over entries [starts, starts + lens), in entry order, all chains at once."""
    order = np.argsort(-lens, kind="stable")
    st, ln = starts[order], lens[order]
    acc = np.zeros((st.size, X.shape[1]), np.float32)
    for j in range(int(ln.max(initial=0))):
        m = int((ln > j).sum())                                   # sorted longest-first: the live chains are a prefix
        pos = st[:m] + j
        x = X[colidx[pos]]
        if keep is not None:
            x = np.where(keep[pos][:, None], x, np.float32(0))
        acc[:m] = O.fmaf32(w[pos][:, None], x, acc[:m])
    out = np.empty_like(acc)
    out[order] = acc
    return out


@pytest.fixture(scope="module")
def sched(dev):
    return _Sched(dev)


def test_regimes(dev, sched):
    """The graph reaches every route: light tasks, CTA-list tasks shorter and longer than MID, split rows, and more light
    tasks than the grid has warps (SMs x 64 at most)."""
    n = (sched.plan["tasks"][:, 2] - sched.plan["tasks"][:, 1]).astype(np.int64)
    lm = sched.A.light_max
    assert ((n > lm) & (n <= MID)).sum() >= 100, f"too few CTA-list tasks of at most {MID} non-zeros"
    assert (n > MID).sum() >= 100, f"too few CTA-list tasks longer than {MID} non-zeros"
    assert (n <= lm).sum() > _sms() * 64, "fewer light tasks than resident warps"
    assert sched.plan["n_split"] >= 6 and sched.plan["longest_row"] >= 5000
    assert sched.A.n_cta_tasks == int((n > lm).sum())


CASES = ([(d, lanes, plan) for d in (32, 64, 128, 256) for lanes in _lane_instances(d) for plan in (True, False)]
         + [(d, 0, plan) for d in (96, 192, 384) for plan in (True, False)])


def _run(sched, dev, d, **kw):
    from mmrec_b200 import ops
    X = torch.from_numpy(np.ascontiguousarray(sched.X[:, :d])).to(dev)
    acc_in = torch.from_numpy(np.ascontiguousarray(sched.acc_in[:, :d])).to(dev)
    Y = torch.empty(sched.n_rows, d, device=dev)
    acc = torch.empty_like(Y)
    ops.spmm_raw(sched.A, X, Y=Y, acc_in=acc_in, acc_out=acc, acc_div=ACC_DIV, **kw)
    assert not bool(sched.A.counters.any())
    return Y.cpu().numpy(), acc.cpu().numpy()


def _check(sched, d, ref, got, what):
    Y, acc = got
    want = ref[:, :d]
    O.assert_bits(Y, want, f"{what}: Y")
    O.assert_bits(acc, (sched.acc_in[:, :d] + want) / np.float32(ACC_DIV), f"{what}: (acc_in + Y) / {ACC_DIV}")


@pytest.mark.parametrize("d,lanes,use_plan", CASES)
def test_summation_order(dev, sched, d, lanes, use_plan):
    T = lanes or _default_lanes(d)
    ref = sched.restate(256 // T, use_plan)
    with _Lanes(lanes):
        got = _run(sched, dev, d, use_plan=use_plan)
    _check(sched, d, ref, got, f"d={d} T={T} plan={use_plan}")


@pytest.mark.parametrize("d", [32, 64, 128, 256])
def test_summation_order_edge_keep(dev, sched, d):
    """The edge-keep mask (one float4 per lane): dropped entries are padding, kept ones weigh fl(v * scale)."""
    rng = np.random.default_rng(d)
    keep = rng.random(sched.A.nnz) < 0.7
    k = np.concatenate([keep, np.zeros(-keep.size % 32, bool)]).reshape(-1, 32).astype(np.uint64)
    words = torch.from_numpy((k << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32).view(np.int32)).to(dev)
    scale = 1.0 / 0.7
    ref = sched.restate(256 // min(32, d // 4), True, keep, scale)
    sched._ref.pop((256 // min(32, d // 4), True, True))
    _check(sched, d, ref, _run(sched, dev, d, drop=(words, scale)), f"d={d} edge-keep")


def test_back_to_back_and_graph_replay(dev, sched):
    """The scratch the kernel reuses across launches (split-row counters) is clean after every launch: two launches in a
    row and a CUDA-graph replay (twice) give the same bits as the first eager launch."""
    from mmrec_b200 import ops
    d = 64
    X = torch.from_numpy(np.ascontiguousarray(sched.X[:, :d])).to(dev)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        outs = [torch.empty(sched.n_rows, d, device=dev) for _ in range(3)]
        ops.spmm_raw(sched.A, X, Y=outs[0])
        ops.spmm_raw(sched.A, X, Y=outs[1])
        side.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            ops.spmm_raw(sched.A, X, Y=outs[2])
        for _ in range(2):
            outs[2].zero_()
            g.replay()
            side.synchronize()
            assert torch.equal(outs[2], outs[0])
    torch.cuda.synchronize()
    assert torch.equal(outs[1], outs[0])
    O.assert_bits(outs[0].cpu().numpy(), sched.restate(256 // 16)[:, :d], "d=64 eager")
