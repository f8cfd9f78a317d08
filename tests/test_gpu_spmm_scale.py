"""K1 SpMM (csrc/spmm.cu) and its work plan (csrc/csr.cu) bit for bit at the sizes the models run.

The exact tests of tests/test_gpu_exact_arith.py run on a few hundred rows.  There the persistent grid is larger than the
task list: every CTA runs one heavy task and phase 2 ends in its first sweep.  The graphs here fill the grid:

* G1, clothing-shaped: the symmetric [users; items] adjacency of `synth.make_graph(40000, 23000, 280000)`, 63k rows, and
  its directed user x item block R with R^T (the backward's long item rows);
* G2, one GPU's shard of config 5: 2M users x 125k zipf items, 6.25M interactions, a symmetric adjacency of 2.1M rows,
  12.5M non-zeros and hub rows of ~10^5 non-zeros, d = 128.

Each graph fixture asserts the regimes it reaches instead of trusting its size (`_sweeps`, `_assert_grid_regimes`).  With
256 threads per CTA the grid holds at most SMs x 8 CTAs and SMs x 64 warps, so more CTA tasks than SMs x 8 means some CTA
runs a second heavy task, and more phase-2 slots than SMs x 64 means a second sweep.

Exactness: matrix values are integers times V_SCALE (`oracle.exact_ints`), dense operands are integers, so every product
is exact in fp32 and, where sum |a||x| < 2^22 units per output (asserted on each case's own operands, `_exact_product`),
every partial sum in any order is an integer below 2^22 units.  The reference is float64 on the device through
`torch.sparse` CSR x dense, built from the host arrays (not from the library's CSR), and is exact.  Epilogue operands are
chosen so that `y + acc_in` is exact in fp32 too; the one rounding left is `/ acc_div`, and float64 division rounded to fp32
equals the fp32 division (double rounding is innocuous for / when 53 >= 2 * 24 + 2), so the references are float64
expressions cast once.  The cosine gate rounds in several places and is checked on G1 against `oracle.spmm_epilogue_f32`.

Multi-layer products outgrow the exact range after one layer (magnitudes grow by the hub degree).  They are pinned on
general fp32 data to the sequence of single products, which the exact cases pin to float64.

Dense operands at G2 size are drawn on the device (a seeded torch generator): on the host they would take gigabytes of
int64.  Comparisons run on the device in row blocks; `oracle.assert_bits` names the first differing element of a block
that fails.  Peak device memory stays below `PEAK_BYTES` (the last test checks it).
"""
import numpy as np
import pytest
import torch

from oracle import mmrec_oracle as O

pytestmark = pytest.mark.gpu

V_SCALE = 2.0 ** -3                 # matrix values: integers in [-3, 3] \ {0} times V_SCALE
X_BITS = 3                          # dense operands: integers with |x| < 2^X_BITS
ACC_BITS = 20                       # acc_in / y_old: |a| < 2^20 units of V_SCALE, so y + a < 2^23 units: exact in fp32
PEAK_BYTES = 10 << 30


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    torch.cuda.init()
    torch.cuda.reset_peak_memory_stats(0)
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ======================================================================================================================
# the plan, restated in numpy
# ======================================================================================================================
def plan_np(rowptr, seg, light_max):
    """`mmrec_spmm_plan` from the row pointer: a row of len <= seg is one task, a longer one ceil(len / seg) segments of
    seg non-zeros (the last one shorter) that share one `split_rows` record {first_slot, n_seg, row_begin, seg}; tasks
    (row, begin, end, split id or -1) in row order are stably sorted by seg - len (longest first), the padding behind
    them.  Tasks longer than light_max are the CTA tasks, a prefix of the sorted list."""
    rowptr = np.asarray(rowptr, np.int64)
    lens = np.diff(rowptr)
    nt = np.where(lens <= seg, 1, -(-lens // seg))
    split = nt > 1
    t_off = np.concatenate([[0], np.cumsum(nt)])
    s_off = np.concatenate([[0], np.cumsum(split)])
    l_off = np.concatenate([[0], np.cumsum(np.where(split, nt, 0))])
    n_tasks = int(t_off[-1])
    row = np.repeat(np.arange(lens.size), nt)
    b = rowptr[row] + (np.arange(n_tasks) - t_off[row]) * seg
    e = np.where(split[row], np.minimum(b + seg, rowptr[row + 1]), rowptr[row + 1])
    sid = np.where(split[row], s_off[row], -1)
    order = np.argsort(seg - (e - b), kind="stable")
    sr = np.nonzero(split)[0]
    return dict(tasks=np.stack([row, b, e, sid], 1)[order].astype(np.int32),
                split_rows=np.stack([l_off[sr], nt[sr], rowptr[sr], np.full(sr.size, seg)], 1).astype(np.int32),
                n_tasks=n_tasks, n_split=int(sr.size), n_slots=int(l_off[-1]), longest_row=int(lens.max(initial=0)),
                n_cta_tasks=int(((e - b) > light_max).sum()))


def _default_lanes(d):
    return d // 12 if d % 3 == 0 else min(32, d // 4)


def _sweeps(A, lanes, use_plan=True):
    """Phase-2 sweeps of the grid at its largest (SMs x 64 warps), for `lanes` lanes per task: a lower bound."""
    light = A.n_tasks - A.n_cta_tasks if use_plan else A.n_rows
    slots = -(-light // (32 // lanes))
    return -(-slots // (_sms() * 64))


def _assert_grid_regimes(A, what, split=True):
    assert A.n_cta_tasks > _sms() * 8, f"{what}: {A.n_cta_tasks} CTA tasks do not give any CTA a second one"
    if split:
        assert A.n_split >= 100, f"{what}: only {A.n_split} split rows"
        assert A.longest_row >= 64 * A.seg, f"{what}: the longest row has {A.longest_row} non-zeros, < 64 segments"


# ======================================================================================================================
# graphs
# ======================================================================================================================
def _ref_csr(dev, rowptr, cols, vals, shape):
    """float64 torch CSRs of the matrix and of its absolute values, from host arrays (values in units)."""
    crow, col = torch.from_numpy(np.asarray(rowptr, np.int64)).to(dev), torch.from_numpy(np.asarray(cols, np.int64)).to(dev)
    v = torch.from_numpy(np.asarray(vals, np.float64)).to(dev)
    return torch.sparse_csr_tensor(crow, col, v, size=shape), torch.sparse_csr_tensor(crow, col, v.abs(), size=shape)


class _Graph:
    """The symmetric [users; items] adjacency of the de-duplicated interactions (u, i) with one integer value per
    interaction on both of its entries (symmetric bit for bit, as the edge-keep mask's transpose needs), as host CSR
    arrays, the library's CSR (built from the unsorted COO) and a float64 reference.  R / Rt: the user x item block."""

    def __init__(self, dev, name, u, i, n_users, n_items, seed):
        from mmrec_b200 import graph
        from mmrec_b200.ops import CSR
        key = graph.unique_sorted(np.asarray(u, np.int64) * n_items + np.asarray(i, np.int64))
        self.u, self.i = key // n_items, key % n_items
        self.name, self.n_users, self.n_items = name, n_users, n_items
        n = self.n = n_users + n_items
        rng = np.random.default_rng(seed)
        w = O.exact_ints(rng, self.u.shape, 2)
        w[w == 0] = 1
        self.w = w
        rows = np.concatenate([self.u, self.i + n_users])
        cols = np.concatenate([self.i + n_users, self.u])
        vals = np.concatenate([w, w])
        order = np.argsort(rows * n + cols, kind="stable")
        self.rows, self.cols, self.vals = rows[order], cols[order], vals[order]
        self.rowptr = np.concatenate([[0], np.cumsum(np.bincount(rows, minlength=n))])
        self.nnz = rows.size
        f32 = lambda v: torch.from_numpy(O.to_f32_exact(v, V_SCALE)).to(dev)
        self.A = CSR.from_coo(torch.from_numpy(rows).to(dev), torch.from_numpy(cols).to(dev), f32(vals), n, n,
                              sum_duplicates=False, symmetric=True)
        assert self.A.nnz == self.nnz
        assert np.array_equal(self.A.rowptr.cpu().numpy(), self.rowptr), f"{name}: rowptr"
        assert np.array_equal(self.A.colidx[:self.nnz].cpu().numpy(), self.cols), f"{name}: column indices"
        O.assert_bits(self.A.vals[:self.nnz], O.to_f32_exact(self.vals, V_SCALE), f"{name}: values")
        self.ref, self.ref_abs = _ref_csr(dev, self.rowptr, self.cols, self.vals, (n, n))
        # R (users x items) and, from its transpose as the library builds it, R^T
        self.R = CSR.from_coo(torch.from_numpy(self.u).to(dev), torch.from_numpy(self.i).to(dev), f32(w), n_users, n_items,
                              sum_duplicates=False, symmetric=False)
        self.Rt = self.R.t()
        ut = np.argsort(self.i * n_users + self.u, kind="stable")
        rp = np.concatenate([[0], np.cumsum(np.bincount(self.u, minlength=n_users))])
        rpt = np.concatenate([[0], np.cumsum(np.bincount(self.i, minlength=n_items))])
        self.R_ref, self.R_ref_abs = _ref_csr(dev, rp, self.i, w, (n_users, n_items))
        self.Rt_ref, self.Rt_ref_abs = _ref_csr(dev, rpt, self.u[ut], w[ut], (n_items, n_users))


def _regimes(G):
    A, Rt = G.A, G.Rt
    return (f"{G.name}: {A.n_rows} rows, nnz {A.nnz}, n_cta_tasks {A.n_cta_tasks}, n_split {A.n_split}, n_slots {A.n_slots}, "
            f"longest_row {A.longest_row} ({-(-A.longest_row // A.seg)} segments), phase-2 sweeps (T=2..32) "
            f"{[_sweeps(A, t) for t in (2, 4, 8, 16, 32)]}; R^T: n_cta_tasks {Rt.n_cta_tasks}, n_split {Rt.n_split}, "
            f"longest_row {Rt.longest_row}")


@pytest.fixture(scope="module")
def g1(dev):
    from mmrec_b200.utils import synth
    s = synth.make_graph(40000, 23000, 280000, seed=0)
    G = _Graph(dev, "G1", *s.train, 40000, 23000, seed=11)
    print(_regimes(G))
    # 63k rows: some CTA runs two heavy tasks and phase 2 sweeps twice at the default lanes; its ~30 split rows of at most
    # ~15 segments leave the split-row regime to G2
    _assert_grid_regimes(G.A, "G1", split=False)
    _assert_grid_regimes(G.Rt, "G1 R^T", split=False)
    return G


@pytest.fixture(scope="module")
def g2(dev):
    from mmrec_b200.utils import synth
    rng = np.random.default_rng(5)
    n_users, n_items, n_edges = 2_000_000, 125_000, 6_250_000
    G = _Graph(dev, "G2", rng.integers(0, n_users, n_edges), synth.zipf_items(rng, n_items, n_edges), n_users, n_items, seed=12)
    print(_regimes(G))
    _assert_grid_regimes(G.A, "G2")
    _assert_grid_regimes(G.Rt, "G2 R^T")
    return G


@pytest.fixture(scope="module")
def graphs(g1, g2):
    return {"G1": g1, "G2": g2}


# ======================================================================================================================
# operands, exact products, comparisons
# ======================================================================================================================
def _ints(dev, shape, bits, seed):
    """float32 integers uniform in (-2^bits, 2^bits), on the device."""
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.empty(shape, dtype=torch.float32, device=dev).random_(1 - (1 << bits), 1 << bits, generator=g)


def _exact_product(M, M_abs, X, vmax=3):
    """M X (M in units of V_SCALE, X integers) as fp32, exact: asserts max|v| max|x| < 2^24 and sum |a||x| < 2^22 units
    for every output, then computes in float64, 32 columns at a time."""
    assert vmax * int(X.abs().max()) < (1 << 24)
    out = torch.empty(M.shape[0], X.shape[1], dtype=torch.float32, device=X.device)
    for c in range(0, X.shape[1], 32):
        xb = X[:, c:c + 32].double()
        s = int((M_abs @ xb.abs()).max())
        assert s < O.EXACT_BUDGET, f"exactness precondition broken: sum |a||x| = {s} units"
        out[:, c:c + 32] = (M @ xb).mul_(V_SCALE)
    return out


def _same(got, what, want, block=1 << 15):
    """got == want(r0, r1) for every block of rows, on the device; a failing block goes to `oracle.assert_bits`."""
    for r0 in range(0, got.shape[0], block):
        r1 = min(got.shape[0], r0 + block)
        w = want(r0, r1)
        if not torch.equal(got[r0:r1], w):
            O.assert_bits(got[r0:r1], w, f"{what} (rows {r0}..{r1})")


def _want_acc(y, a, div):
    """fl32((y + a) / div) for y + a exact in fp32 (see the module docstring)."""
    def f(r0, r1):
        s = y[r0:r1].double()
        if a is not None:
            s += a[r0:r1].double()
        return (s / div).float() if div != 1.0 else s.float()
    return f


class _Operands:
    """X, the exact product y = A X and acc_in for one (matrix, d), kept for the tests that follow (one set at a time:
    at G2 and d = 256 each tensor is 2.2 GB).  `acc_in_is_x`: acc_in is X itself, the first layer of `propagate_mean`
    (acc_in = E_0 = X), one tensor fewer; |x| < 2^X_BITS keeps y + x exact."""
    key, val = None, None

    @classmethod
    def get(cls, dev, key, seed, M, M_abs, n_cols, d, acc_in_is_x=False):
        if cls.key != key:
            cls.release()
            X = _ints(dev, (n_cols, d), X_BITS, seed)
            y = _exact_product(M, M_abs, X)
            acc_in = X if acc_in_is_x else _ints(dev, (M.shape[0], d), ACC_BITS, seed + 1).mul_(V_SCALE)
            cls.key, cls.val = key, (X, y, acc_in)
        return cls.val

    @classmethod
    def release(cls):
        cls.key = cls.val = None
        torch.cuda.empty_cache()


def _forms(A, X, y, acc_in, what, use_plan=True, drop=None):
    """Every epilogue of one product against the exact y: Y; acc_out with acc_in and acc_div 1 and 3; acc_out / 3 without
    acc_in; Y += A X (not with the edge-keep mask).  The split-row counters are zero after every call."""
    from mmrec_b200 import ops
    n, d = y.shape

    def run(**kw):
        ops.spmm_raw(A, X, use_plan=use_plan, drop=drop, **kw)
        assert not bool(A.counters.any()), f"{what}: split-row counters left nonzero"

    out = torch.full((n, d), 7.0, device=y.device)
    run(Y=out)
    _same(out, f"{what} Y", lambda r0, r1: y[r0:r1])
    for div in (1.0, 3.0):
        out.fill_(7.0)
        run(acc_in=acc_in, acc_out=out, acc_div=div)
        _same(out, f"{what} acc_out (acc_div {div})", _want_acc(y, acc_in, div))
    run(acc_out=out, acc_div=3.0)
    _same(out, f"{what} acc_out / 3 without acc_in", _want_acc(y, None, 3.0))
    if drop is None:
        out.copy_(acc_in)
        run(Y=out, y_accumulate=True)
        _same(out, f"{what} Y += AX", _want_acc(y, acc_in, 1.0))
    del out


class _Lanes:
    def __init__(self, lanes):
        from mmrec_b200 import _lib
        self.lib, self.lanes = _lib.load(), lanes

    def __enter__(self):
        from mmrec_b200 import _lib
        _lib.check(self.lib.mmrec_spmm_set_lanes(self.lanes), "mmrec_spmm_set_lanes")

    def __exit__(self, *exc):
        self.lib.mmrec_spmm_set_lanes(0)


# ======================================================================================================================
# 1. the plan, bit for bit
# ======================================================================================================================
@pytest.mark.parametrize("seg,light_max", [(None, None), (32, None), (4000, None), (None, 1), (None, 4000)])
def test_plan_bit_for_bit_g2(dev, g2, seg, light_max):
    """`mmrec_spmm_plan` on G2 against its numpy restatement at the default and at the limits of seg and light_max, and an
    exact product on each plan (light_max 1: every task of more than one non-zero in phase 1; 4000: none; seg 32: every
    row longer than 32 split)."""
    from mmrec_b200 import ops
    from mmrec_b200.ops import CSR
    _Operands.release()
    G = g2
    if seg is None and light_max is None:
        A = G.A
    else:
        r, c, v = G.A.coo()
        A = CSR.from_coo(r, c, v, G.n, G.n, sum_duplicates=False, symmetric=True, seg=seg, light_max=light_max)
    s, lm = A.seg, A.light_max
    assert (s, lm) == (seg or ops.SEG, light_max or ops.LIGHT_MAX)
    want = plan_np(G.rowptr, s, lm)
    what = f"G2 plan seg={s} light_max={lm}"
    for k in ("n_tasks", "n_split", "n_slots", "longest_row", "n_cta_tasks"):
        assert getattr(A, k) == want[k], f"{what}: {k} {getattr(A, k)} != {want[k]}"
    tasks = A.tasks.view(-1, 4)[:A.n_tasks].cpu().numpy()
    bad = np.nonzero((tasks != want["tasks"]).any(1))[0]
    assert bad.size == 0, f"{what}: {bad.size} task records differ, first at {bad[0]}: {tasks[bad[0]]} != {want['tasks'][bad[0]]}"
    split = A.split_rows.view(-1, 4)[:A.n_split].cpu().numpy()
    bad = np.nonzero((split != want["split_rows"]).any(1))[0]
    assert bad.size == 0, f"{what}: {bad.size} split records differ, first at {bad[0]}: {split[bad[0]]} != {want['split_rows'][bad[0]]}"
    X = _ints(dev, (G.n, 32), X_BITS, 99)
    y = _exact_product(G.ref, G.ref_abs, X)
    out = torch.empty_like(y)
    ops.spmm_raw(A, X, Y=out)
    assert not bool(A.counters.any())
    _same(out, f"{what}: Y", lambda r0, r1: y[r0:r1])


# ======================================================================================================================
# 2, 3. one product, every epilogue, every lane count, with and without the plan; the widths 3d on G1
# ======================================================================================================================
def _lane_instances(d):
    """0 (the default, one float4 per lane) and the override's other instances, 2 and 4 float4 per lane (at d = 256 the
    default has 32 lanes already, and 2 float4 per lane is the override's 32)."""
    return [0] + [t for t in (min(32, d // 8), min(32, d // 16)) if t != min(32, d // 4)]


PRODUCT_CASES = ([(g, d, lanes, plan) for g in ("G1", "G2") for d in (32, 64, 128, 256) for lanes in _lane_instances(d)
                  for plan in (True, False)]
                 + [("G1", d, 0, plan) for d in (96, 192, 384) for plan in (True, False)])


@pytest.mark.parametrize("graph,d,lanes,use_plan", PRODUCT_CASES)
def test_product_every_epilogue(dev, graphs, graph, d, lanes, use_plan):
    G = graphs[graph]
    # G2: acc_in = X (the peak stays below PEAK_BYTES at d = 256); G1 keeps an acc_in of its own, so that reading X where
    # acc_in belongs fails there
    X, y, acc_in = _Operands.get(dev, (graph, d), 100 * int(graph[1]) + d, G.ref, G.ref_abs, G.n, d, acc_in_is_x=graph == "G2")
    T = lanes or _default_lanes(d)
    if graph == "G2" or lanes == 0:            # G1 with 2 or 4 lanes per task fits phase 2 in one sweep; G2 covers those
        assert _sweeps(G.A, T, use_plan) >= 2, f"{graph} d={d} T={T}: phase 2 in one sweep"
    with _Lanes(lanes):
        _forms(G.A, X, y, acc_in, f"{graph} d={d} T={T} plan={use_plan}", use_plan)


# ======================================================================================================================
# 4. the edge-keep mask on G2
# ======================================================================================================================
def test_edge_keep_mask_g2(dev, g2):
    """SelfCF's dropped adjacency on G2 at d = 128: `keep` against float64 on the compacted matrix, the mirrored `keep_t`
    against its transpose.  Scale 2 (keep probability 1/2) keeps every weight fl(v * scale) exact."""
    from mmrec_b200 import graph, ops
    _Operands.release()
    G, d, n = g2, 128, g2.n
    draw_of, mirror = graph.dropout_entry_maps(G.u, G.i, G.n_users, G.n_items)
    draw_of, mirror = torch.from_numpy(draw_of).to(dev), torch.from_numpy(mirror).to(dev)
    draws = torch.rand(G.nnz, generator=torch.Generator(device=dev).manual_seed(3), device=dev)
    keep, keep_t = ops.edge_keep_bits(draws, 0.5, draw_of, mirror)
    e = torch.arange(G.nnz, device=dev)
    unpack = lambda bits: ((bits.long()[e >> 5] >> (e & 31)) & 1).bool()
    kept = torch.floor(0.5 + draws[draw_of.long()]) != 0             # the keep rule in fp32, independent of the kernel
    assert torch.equal(unpack(keep), kept) and torch.equal(unpack(keep_t), kept[mirror.long()])
    del e, draws
    rows = torch.from_numpy(G.rows).to(dev)
    cols = torch.from_numpy(G.cols).to(dev)
    vals = torch.from_numpy(G.vals).to(dev, torch.float64) * 2.0     # units of V_SCALE, times the scale
    X = _ints(dev, (n, d), X_BITS, 41)
    acc_in = _ints(dev, (n, d), ACC_BITS, 42).mul_(V_SCALE)
    for bits, (r, c) in ((keep, (rows, cols)), (keep_t, (cols, rows))):
        r, c, v = r[kept], c[kept], vals[kept]
        order = torch.argsort(r * n + c)                               # the compacted matrix (its transpose for keep_t)
        r, c, v = r[order], c[order], v[order]
        crow = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.bincount(r, minlength=n).cumsum(0)])
        M = torch.sparse_csr_tensor(crow, c, v, size=(n, n))
        M_abs = torch.sparse_csr_tensor(crow, c, v.abs(), size=(n, n))
        y = _exact_product(M, M_abs, X, vmax=6)
        del r, c, v, order, M, M_abs
        _forms(G.A, X, y, acc_in, f"G2 {'keep_t' if bits is keep_t else 'keep'}", drop=(bits, 2.0))
        del y


# ======================================================================================================================
# 5. the backward: R^T
# ======================================================================================================================
@pytest.mark.parametrize("graph,d", [("G1", 64), ("G2", 128)])
def test_backward_transpose(dev, graphs, graph, d):
    """`ops.spmm` on R and its autograd backward on R^T (the transpose the library builds; item rows of up to 10^5
    non-zeros at G2), then every epilogue on R^T."""
    from mmrec_b200 import ops
    _Operands.release()
    G = graphs[graph]
    X = _ints(dev, (G.n_items, d), X_BITS, 51).requires_grad_(True)
    g = _ints(dev, (G.n_users, d), X_BITS, 52)
    y = ops.spmm(G.R, X)
    yr = _exact_product(G.R_ref, G.R_ref_abs, X.detach())
    _same(y.detach(), f"{graph} R X", lambda r0, r1: yr[r0:r1])
    y.backward(g)
    assert not bool(G.Rt.counters.any())
    gx = _exact_product(G.Rt_ref, G.Rt_ref_abs, g)
    _same(X.grad, f"{graph} R^T g (autograd)", lambda r0, r1: gx[r0:r1])
    del X, y, yr
    acc_in = _ints(dev, (G.n_items, d), ACC_BITS, 53).mul_(V_SCALE)
    _forms(G.Rt, g, gx, acc_in, f"{graph} R^T")


# ======================================================================================================================
# 6. multi-layer routes, pinned to the single products
# ======================================================================================================================
def _mm_graph(dev, n_items, k, seed):
    """A FREEDOM-like item-item graph: k random neighbours per item, general fp32 weights."""
    from mmrec_b200.ops import CSR
    g = torch.Generator(device=dev).manual_seed(seed)
    row = torch.arange(n_items, device=dev).repeat_interleave(k)
    col = torch.randint(0, n_items, (n_items * k,), generator=g, device=dev)
    val = torch.rand(n_items * k, generator=g, device=dev) / k
    return CSR.from_coo(row, col, val, n_items, n_items)


@pytest.mark.parametrize("post", [False, True])
@pytest.mark.parametrize("cooperative", [True, False])
def test_propagate_mean_fused_g2(dev, g2, cooperative, post):
    """Config 5's inference route: `propagate_mean_fused` from the (user table, item table) pair, two layers, with and
    without FREEDOM's `+ mm_adj @ item table` on the item rows, bit for bit against `_propagate_mean_post_unfused` (one
    `spmm_raw` per product) on general fp32 data at d = 128."""
    from mmrec_b200 import ops
    _Operands.release()
    G, d = g2, 128
    g = torch.Generator(device=dev).manual_seed(61)
    ut = torch.randn(G.n_users, d, generator=g, device=dev)
    it = torch.randn(G.n_items, d, generator=g, device=dev)
    M = _mm_graph(dev, G.n_items, 10, 62) if post else None
    kw = dict(post_csr=M, post_x=it if post else None, post_row0=G.n_users)
    before = ops.launch_count()
    got = ops.propagate_mean_fused(G.A, (ut, it), 2, cooperative=cooperative, **kw)
    assert ops.launch_count() - before == (1 if cooperative else 2), "the chained kernel did not take this shape"
    assert not bool(G.A.counters.any())
    want = ops._propagate_mean_post_unfused(G.A, torch.cat([ut, it]), 2, kw["post_csr"], kw["post_x"], 1, G.n_users)
    _same(got, f"propagate_mean_fused cooperative={cooperative} post={post}", lambda r0, r1: want[r0:r1])


def test_propagate_mean_backward_g2(dev, g2):
    """`propagate_mean`'s backward (g_l = g / (L + 1) + A^T g_{l+1}) against the same single `spmm_raw` calls, G2, d = 128."""
    from mmrec_b200 import ops
    _Operands.release()
    G, d, L = g2, 128, 3
    g = torch.Generator(device=dev).manual_seed(71)
    ego = torch.randn(G.n, d, generator=g, device=dev).requires_grad_(True)
    up = torch.randn(G.n, d, generator=g, device=dev)
    ops.propagate_mean(G.A, ego, L).backward(up)
    gm = up / (L + 1)
    cur = gm
    for _ in range(L):
        nxt = torch.empty_like(gm)
        ops.spmm_raw(G.A.t(), cur, acc_in=gm, acc_out=nxt)
        cur = nxt
    _same(ego.grad, "propagate_mean backward", lambda r0, r1: cur[r0:r1])


# ======================================================================================================================
# 7. PanelCSR at its default panel size
# ======================================================================================================================
def test_panel_csr_default_panels_g2(dev, g2):
    """Config 5's column-panelled product at the default `panel_bytes` (d = 128: ~22 panels): Y accumulated over the
    panels, and the running sum with the division on the last one, exact."""
    from mmrec_b200 import ops
    G, d = g2, 128
    X, y, acc_in = _Operands.get(dev, ("G2", d), 200 + d, G.ref, G.ref_abs, G.n, d, acc_in_is_x=True)
    r, c, v = G.A.coo()
    P = ops.PanelCSR.from_coo(r, c, v, G.n, G.n, d, sum_duplicates=False, symmetric=True)
    del r, c, v
    assert len(P.panels) >= 20, len(P.panels)
    Y, out = torch.full((G.n, d), 7.0, device=dev), torch.full((G.n, d), 7.0, device=dev)
    ops.spmm_raw(P, X, Y=Y, acc_in=acc_in, acc_out=out, acc_div=3.0)
    assert not any(bool(p.counters.any()) for p in P.panels)
    _same(Y, "PanelCSR Y", lambda r0, r1: y[r0:r1])
    _same(out, "PanelCSR acc_out / 3", _want_acc(y, acc_in, 3.0))


# ======================================================================================================================
# 8. LayerGCN's cosine gate at scale
# ======================================================================================================================
def test_cosine_gate_g1(dev, g1):
    """The gate on G1 at d = 64 with X in {-1, 0, 1}: y, y.x, |y|^2 and |x|^2 exact (asserted as `_SpmmCase` does), so the
    gated rows equal `oracle.spmm_epilogue_f32` bit for bit.  `propagate_layergcn` (one layer, gate_ref = E_0) and the
    gate on Y and on a running sum."""
    from mmrec_b200 import ops
    _Operands.release()
    G, d = g1, 64
    X = _ints(dev, (G.n, d), 1, 81)
    y = _exact_product(G.ref, G.ref_abs, X).cpu().numpy()
    x = X.cpu().numpy()
    yi = np.abs(y.astype(np.float64) / V_SCALE)
    assert float((yi * np.abs(x)).sum(1).max()) < O.EXACT_BUDGET and float((yi * yi).sum(1).max()) < O.EXACT_BUDGET
    assert float((x * x).sum(1).max()) < O.EXACT_BUDGET
    got = ops.propagate_layergcn(G.A, X, 1)
    O.assert_bits(got, O.spmm_epilogue_f32(y, None, 1.0, gate_ref=x)[1], "G1 propagate_layergcn, one layer")
    acc_in = _ints(dev, (G.n, d), ACC_BITS, 82).mul_(V_SCALE)
    Y, out = torch.empty(G.n, d, device=dev), torch.empty(G.n, d, device=dev)
    ops.spmm_raw(G.A, X, Y=Y, acc_in=acc_in, acc_out=out, gate_ref=X)
    wy, wa = O.spmm_epilogue_f32(y, acc_in.cpu().numpy(), 1.0, gate_ref=x)
    O.assert_bits(Y, wy, "G1 gated Y")
    O.assert_bits(out, wa, "G1 gated acc_out")


# ======================================================================================================================
# 9. run to run
# ======================================================================================================================
def test_run_to_run_g2(dev, g2):
    """Two calls on general fp32 operands give the same bits: the split rows' segment-order reduction does not depend on
    which segment arrives last."""
    from mmrec_b200 import ops
    _Operands.release()
    G, d = g2, 128
    g = torch.Generator(device=dev).manual_seed(91)
    X = torch.randn(G.n, d, generator=g, device=dev)
    acc_in = torch.randn(G.n, d, generator=g, device=dev)
    outs = []
    for _ in range(2):
        Y, acc = torch.empty(G.n, d, device=dev), torch.empty(G.n, d, device=dev)
        ops.spmm_raw(G.A, X, Y=Y, acc_in=acc_in, acc_out=acc, acc_div=3.0)
        outs.append((Y, acc))
    _same(outs[0][0], "run to run Y", lambda r0, r1: outs[1][0][r0:r1])
    _same(outs[0][1], "run to run acc_out", lambda r0, r1: outs[1][1][r0:r1])


def test_peak_device_memory(dev):
    """The file's peak stays below PEAK_BYTES (the GPUs are shared)."""
    _Operands.release()
    peak = torch.cuda.max_memory_allocated(0)
    print(f"peak device memory: {peak / 2 ** 30:.2f} GiB")
    assert peak < PEAK_BYTES, f"peak {peak / 2 ** 30:.2f} GiB"
