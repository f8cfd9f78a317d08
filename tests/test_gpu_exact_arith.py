"""K1 SpMM, K2 projection, K3t unfused scoring, K5 training kernels and the Adam step, bit for bit.

Most tests of these kernels compare one Frobenius norm per tensor with a CPU result.  An error confined to a few
elements -- one ragged tile, one K split, the tail segment of a split row, one lane width, a 3xTF32 kernel that loses a
compensation term on some tiles -- hides in such a norm.  The tests here feed operands on which every correct kernel
returns one result, bit for bit, and compare with `torch.equal`:

* Operands are integers times a power of two (`oracle.exact_ints`).  If every product is exact in fp32 and, for each
  output, sum |a||b| < 2^22 in units of the product granularity (`oracle.assert_exact_matmul`, asserted in every test),
  each partial sum of any summation order is an integer below 2^22 units.  ASSUMPTION (as for the kNN build, K7): the fp32
  adder -- CUDA cores or the tensor cores' accumulator -- keeps at least 24 significant bits after aligning its operands,
  so such a sum is never rounded.  K splits, chunk rotations, lane widths and tilings then cannot change a bit.
* 3xTF32 (K2 "tc", K3t "tc"): one operand carries 12-13 significant bits, so its tf32 `lo` part is nonzero and exact, the
  other has at most 11 bits (`lo` = 0).  A missing `lo.hi` or `hi.lo` term is then a wrong integer.  Every K2 / K3t case
  runs twice: low bits on the left operand, then on the right one.
* Epilogues that round (`/ acc_div`, `+ post`, LayerGCN's cosine gate, the row L2 norm) are emulated in numpy float32
  (`oracle.spmm_epilogue_f32`, `oracle.l2_rows_f32`): their inputs are exact and each step is one IEEE rounding (the
  library is compiled without --use_fast_math, so `/` and `sqrtf` are IEEE).
* Adam is elementwise: `oracle.adam_foreach_f32` restates torch's foreach Adam with its FMAs, and the kernels are compared
  bit for bit with it and with `torch.optim.Adam(foreach=True)` on the device.

The tensor-core paths are also checked for precision on positive full-mantissa operands, element by element, against
the worst-case bound derived in `test_tf32_paths_per_element_bound`.
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import mmrec_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


# ======================================================================================================================
# K1: SpMM
# ======================================================================================================================
SEG = 512
# row lengths: empty rows, a lane-group row, 33 (first CTA-sized task), one full segment, 513 / 520 (two segments; the
# 8-non-zero tail of 520 is light enough for the lane-group phase while its first segment runs in the CTA phase) and
# 4200 = 8 x 512 + 104 (nine segments: the second batch of spmm_split_finish's 8-partial loop)
ROW_LENS = [0, 0, 1, 7, 32, 33, 64, 511, 512, 513, 520, 4200, 0, 3]
N_COLS = 4500


def _spmm_matrix(seed, n_fill=300):
    rng = np.random.default_rng(seed)
    lens = ROW_LENS + list(rng.integers(0, 40, n_fill))
    rows, cols = [], []
    for r, n in enumerate(lens):
        rows.append(np.full(n, r, dtype=np.int64))
        cols.append(np.sort(rng.choice(N_COLS, size=n, replace=False)).astype(np.int64))
    row, col = np.concatenate(rows), np.concatenate(cols)
    vals = O.exact_ints(rng, row.shape, 2) + 0                       # |v| <= 3, units of 1/8
    vals[vals == 0] = 1
    return len(lens), row, col, vals


def _csr_int(n_rows, n_cols, row, col, vals):
    import scipy.sparse as sp
    return sp.csr_matrix((vals.astype(np.int64), (row, col)), shape=(n_rows, n_cols))


V_SCALE, X_SCALE = 2.0 ** -3, 2.0 ** -1


def _spmm_exact(Ai, Xi):
    """Exact integer product (units V_SCALE * X_SCALE) after asserting the exactness precondition."""
    absA = abs(Ai)
    s = int((absA @ np.abs(Xi)).max(initial=0))
    assert int(np.abs(Xi).max(initial=0)) * int(absA.max()) < (1 << 24)
    assert s < O.EXACT_BUDGET, s
    return Ai @ Xi


class _SpmmCase:
    def __init__(self, dev, d, seed=1):
        from mmrec_b200.ops import CSR
        self.n, row, col, vals = _spmm_matrix(seed)
        rng = np.random.default_rng(seed + d)
        self.Ai = _csr_int(self.n, N_COLS, row, col, vals)
        self.Xi = O.exact_ints(rng, (N_COLS, d), 1)                      # |x| <= 1: the gate's |y|^2 stays exact at d = 256
        self.Yi = _spmm_exact(self.Ai, self.Xi)
        self.y = O.to_f32_exact(self.Yi, V_SCALE * X_SCALE)
        self.acc_in = O.to_f32_exact(O.exact_ints(rng, (self.n, d), 10), V_SCALE * X_SCALE)
        self.post = O.to_f32_exact(O.exact_ints(rng, (self.n, d), 6), 2.0 ** -7)
        # gate: dot, |y|^2 and |ref|^2 must be exact integers (units V X, V^2 X^2, 1)
        self.ref = O.exact_ints(rng, (self.n, d), 3)
        ui = np.abs(self.Yi)
        assert int((ui * np.abs(self.ref)).sum(1).max()) < O.EXACT_BUDGET and int((ui * ui).sum(1).max()) < O.EXACT_BUDGET
        assert int((self.ref * self.ref).sum(1).max()) < O.EXACT_BUDGET
        self.ref = O.to_f32_exact(self.ref, 1.0)
        self.X = torch.from_numpy(O.to_f32_exact(self.Xi, X_SCALE)).to(dev)
        self.A = CSR.from_coo(torch.from_numpy(row).to(dev), torch.from_numpy(col).to(dev),
                              torch.from_numpy(O.to_f32_exact(vals, V_SCALE)).to(dev), self.n, N_COLS)
        assert self.A.nnz == row.size and self.A.longest_row == 4200 and self.A.n_split == 3      # rows of 513, 520 and 4200


def _run_epilogues(dev, case, use_plan, what):
    from mmrec_b200 import ops
    d = case.X.shape[1]
    n = case.n
    Y = torch.full((n, d), 7.0, device=dev)
    ops.spmm_raw(case.A, case.X, Y=Y, use_plan=use_plan)
    O.assert_bits(Y, case.y, f"{what} Y")
    acc_in = torch.from_numpy(case.acc_in).to(dev)
    post = torch.from_numpy(case.post).to(dev)
    for div in (1.0, 4.0, 3.0):
        out = torch.full((n, d), 7.0, device=dev)
        Y2 = torch.empty(n, d, device=dev)
        ops.spmm_raw(case.A, case.X, Y=Y2, acc_in=acc_in, acc_out=out, acc_div=div, use_plan=use_plan)
        _, want = O.spmm_epilogue_f32(case.y, case.acc_in, div)
        O.assert_bits(out, want, f"{what} acc_out (acc_div {div})")
        O.assert_bits(Y2, case.y, f"{what} Y beside acc_out")
    out = torch.empty(n, d, device=dev)                              # acc_out without acc_in, divided
    ops.spmm_raw(case.A, case.X, acc_out=out, acc_div=3.0, use_plan=use_plan)
    O.assert_bits(out, O.spmm_epilogue_f32(case.y, None, 3.0)[1], f"{what} acc_out / 3 without acc_in")
    # LayerGCN's gate on Y and on the running sum
    ref = torch.from_numpy(case.ref).to(dev)
    Yg, accg = torch.empty(n, d, device=dev), torch.empty(n, d, device=dev)
    ops.spmm_raw(case.A, case.X, Y=Yg, acc_in=acc_in, acc_out=accg, gate_ref=ref, use_plan=use_plan)
    wy, wa = O.spmm_epilogue_f32(case.y, case.acc_in, 1.0, gate_ref=case.ref)
    O.assert_bits(Yg, wy, f"{what} gated Y")
    O.assert_bits(accg, wa, f"{what} gated acc_out")
    # Y += A X (y_accumulate) with a running sum
    Ya = torch.from_numpy(case.acc_in).to(dev).clone()
    outa = torch.empty(n, d, device=dev)
    ops.spmm_raw(case.A, case.X, Y=Ya, acc_in=acc_in, acc_out=outa, acc_div=3.0, use_plan=use_plan, y_accumulate=True)
    wy, wa = O.spmm_epilogue_f32(case.y, case.acc_in, 3.0, y_old=case.acc_in)
    O.assert_bits(Ya, wy, f"{what} Y += AX")
    O.assert_bits(outa, wa, f"{what} acc_out of the accumulating form")


def _lane_widths(d):
    return sorted({min(32, d // 4), min(32, d // 8), min(32, d // 16)}, reverse=True)


SPMM_VEC = [(d, t) for d in (32, 64, 128, 256) for t in _lane_widths(d)]


@pytest.mark.parametrize("use_plan", [True, False])
@pytest.mark.parametrize("d,lanes", SPMM_VEC)
def test_spmm_vec_every_lane_width_and_epilogue(dev, d, lanes, use_plan):
    """Vector kernel at every (d, lanes per task) instance, with and without the work plan (split rows, CTA tasks)."""
    from mmrec_b200 import _lib
    lib = _lib.load()
    case = _SpmmCase(dev, d)
    assert case.A.n_cta_tasks >= 1
    _lib.check(lib.mmrec_spmm_set_lanes(lanes), "mmrec_spmm_set_lanes")
    try:
        _run_epilogues(dev, case, use_plan, f"d={d} T={lanes} plan={use_plan}")
    finally:
        lib.mmrec_spmm_set_lanes(0)


@pytest.mark.parametrize("d", [5, 48, 100])
def test_spmm_generic_widths(dev, d):
    """Widths without a vector instance run the generic kernel (whole rows, scalar loads)."""
    _run_epilogues(dev, _SpmmCase(dev, d), True, f"generic d={d}")


@pytest.mark.parametrize("use_plan", [True, False])
@pytest.mark.parametrize("d", [96, 192, 384])
def test_spmm_vec_3d_every_epilogue(dev, d, use_plan):
    """The width-3d instances (three float4 per lane, SLMRec's three views side by side), every epilogue: the gate and
    Y += A X included, which reduce or read across the whole 3d row."""
    _run_epilogues(dev, _SpmmCase(dev, d), use_plan, f"3d d={d} plan={use_plan}")


def _spmm_abi(case, d, X, ldx, Y, ldy, acc_in, acc_out, ldacc, acc_div, ref, ldref):
    """`mmrec_spmm_run_f32` with raw addresses and leading dimensions (ops.spmm_raw would copy to contiguous operands)."""
    from mmrec_b200 import _lib
    A = case.A
    op = _lib.SpmmOp(n_rows=A.n_rows, n_cols=A.n_cols, rowptr=A.rowptr.data_ptr(), colidx=A.colidx.data_ptr(), vals=A.vals.data_ptr(),
                     tasks=A.tasks.data_ptr(), n_tasks=A.n_tasks, n_cta_tasks=A.n_cta_tasks, split_rows=A.split_rows.data_ptr(),
                     counters=A.counters.data_ptr(), partial=A.partial(d).data_ptr(), X=X, ldx=ldx, Y=Y, ldy=ldy,
                     acc_in=acc_in, acc_out=acc_out, ldacc=ldacc, acc_div=acc_div, gate_ref=ref, ldgate=ldref)
    _lib.check(_lib.load().mmrec_spmm_run_f32(d, 1, ctypes.byref(op), 0, torch.cuda.current_stream().cuda_stream), "mmrec_spmm_run_f32")


@pytest.mark.parametrize("d,shift", [(64, 1), (128, 2), (32, 0)])
def test_spmm_misaligned_and_strided_through_the_op_descriptor(dev, d, shift):
    """Misaligned X / Y / acc (offset by `shift` floats) and leading dimensions > d reach the generic kernel; shift 0
    with padded rows (ld % 4 == 0, 16-byte aligned) keeps the vector kernel on strided operands."""
    case = _SpmmCase(dev, d)
    n = case.n
    ldx, ldy, ldacc, ldg = d + 4 * (shift == 0) + 3 * (shift > 0), d + 4, d + 8, d + 4 + shift

    def strided(a, ld, sh):
        buf = torch.full((a.shape[0] * ld + 8,), 5.0, device=dev)
        v = buf[sh:sh + a.shape[0] * ld].view(a.shape[0], ld)
        v[:, :a.shape[1]] = torch.as_tensor(a, device=dev)
        return buf, v

    _, Xv = strided(case.X, ldx, shift)
    _, Yv = strided(np.zeros((n, d), np.float32), ldy, shift)
    _, Iv = strided(case.acc_in, ldacc, shift)
    _, Ov = strided(np.zeros((n, d), np.float32), ldacc, shift)
    _, Rv = strided(case.ref, ldg, shift)
    _spmm_abi(case, d, Xv.data_ptr(), ldx, Yv.data_ptr(), ldy, Iv.data_ptr(), Ov.data_ptr(), ldacc, 3.0, Rv.data_ptr(), ldg)
    wy, wa = O.spmm_epilogue_f32(case.y, case.acc_in, 3.0, gate_ref=case.ref)
    O.assert_bits(Yv[:, :d], wy, "strided gated Y")
    O.assert_bits(Ov[:, :d], wa, "strided gated acc_out / 3")
    assert bool((Yv[:, d:] == 5.0).all()) and bool((Ov[:, d:] == 5.0).all()), "wrote past d"


@pytest.mark.parametrize("d", [64, 96])
def test_spmm_transpose(dev, d):
    """The backward CSR (A^T): long columns of A become long rows."""
    from mmrec_b200 import ops
    case = _SpmmCase(dev, d)
    rng = np.random.default_rng(d)
    Gi = O.exact_ints(rng, (case.n, d), 2)
    want = O.to_f32_exact(_spmm_exact(case.Ai.T.tocsr(), Gi), V_SCALE * X_SCALE)
    At = case.A.t()
    out = torch.empty(N_COLS, d, device=dev)
    ops.spmm_raw(At, torch.from_numpy(O.to_f32_exact(Gi, X_SCALE)).to(dev), Y=out)
    O.assert_bits(out, want, "A^T G")


@pytest.mark.parametrize("d", [64, 128])
def test_spmm_panel_csr(dev, d):
    """The accumulating Y (y_accumulate) through PanelCSR: Y and the running sum accumulate over ~5 column panels; the
    division comes with the last one."""
    from mmrec_b200 import ops
    case = _SpmmCase(dev, d)
    r, c, v = case.A.coo()
    P = ops.PanelCSR.from_coo(r, c, v, case.n, N_COLS, d, panel_bytes=1024 * 4 * d)
    assert len(P.panels) >= 4
    Y, out = torch.empty(case.n, d, device=dev), torch.empty(case.n, d, device=dev)
    ops.spmm_raw(P, case.X, Y=Y, acc_in=torch.from_numpy(case.acc_in).to(dev), acc_out=out, acc_div=3.0)
    wy, wa = O.spmm_epilogue_f32(case.y, case.acc_in, 3.0)
    O.assert_bits(Y, wy, "panelled Y")
    O.assert_bits(out, wa, "panelled acc_out / 3")


@pytest.mark.parametrize("d", [32, 64, 256])
def test_spmm_chain_with_post_rows(dev, d):
    """The cooperative chain kernel: mean of E_0..E_2 of a square graph with long rows, then `+ post` on the item rows
    (FREEDOM's `i_g + h`, h = M @ x through one more chained SpMM)."""
    from mmrec_b200 import ops
    from mmrec_b200.ops import CSR
    n, row, col, vals = _spmm_matrix(7, n_fill=N_COLS - len(ROW_LENS))
    assert n == N_COLS
    rng = np.random.default_rng(d)
    Ai = _csr_int(n, n, row, col, vals)
    E0 = O.exact_ints(rng, (n, d), 2)
    E1 = _spmm_exact(Ai, E0)                                         # units V
    E2 = _spmm_exact(Ai, E1)                                         # units V^2
    assert int(np.abs(E2).max()) < (1 << 22)
    n_post, row0 = 1000, n - 1000
    mr = rng.integers(0, n_post, 8000); mc = rng.integers(0, n_post, 8000)
    key = np.unique(mr * n_post + mc)
    mr, mc = key // n_post, key % n_post
    mv = O.exact_ints(rng, mr.shape, 2)
    mv[mv == 0] = 1
    Mi = _csr_int(n_post, n_post, mr, mc, mv)
    xi = O.exact_ints(rng, (n_post, d), 2)
    Hi = _spmm_exact(Mi, xi)
    # acc = ((E0 + E1) + E2) / 3 + h: E0 + E1 and + E2 are exact integer sums (units V^2), one rounding each for / and +
    s = E0 * 64 + E1 * 8 + E2
    assert int(np.abs(s).max()) < (1 << 24)
    h = O.to_f32_exact(Hi, V_SCALE)
    want = O.fdiv_f32(O.to_f32_exact(s, V_SCALE ** 2), 3.0)
    want[row0:] = (want[row0:] + h).astype(np.float32)
    A = CSR.from_coo(torch.from_numpy(row).to(dev), torch.from_numpy(col).to(dev), torch.from_numpy(O.to_f32_exact(vals, V_SCALE)).to(dev), n, n)
    M = CSR.from_coo(torch.from_numpy(mr).to(dev), torch.from_numpy(mc).to(dev), torch.from_numpy(O.to_f32_exact(mv, V_SCALE)).to(dev),
                     n_post, n_post)
    ego = torch.from_numpy(O.to_f32_exact(E0, 1.0)).to(dev)
    before = ops.launch_count()
    got = ops.propagate_mean_fused(A, ego, 2, post_csr=M, post_x=torch.from_numpy(O.to_f32_exact(xi, 1.0)).to(dev), post_row0=row0)
    assert ops.launch_count() - before == 1, "the chained kernel did not take this shape"
    O.assert_bits(got, want, "chained mean + post")


# ======================================================================================================================
# K2: projection
# ======================================================================================================================
def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pj_splits(n_out, F, d):
    """`pj_plan` of csrc/project_tc.cu: (K splits, chunks per split, chunks of the last split)."""
    n_chunks = -(-F // 32)
    n_tiles = -(-n_out // 128)
    splits = max(1, _sm_count() // n_tiles)
    if splits > n_chunks // 4:
        splits = n_chunks // 4 if n_chunks // 4 > 0 else 1
    splits = min(splits, 32)
    cps = -(-n_chunks // splits)
    n_splits = -(-n_chunks // cps)
    return n_splits, cps, n_chunks - (n_splits - 1) * cps


# (n_out, F, d, K splits): every N = 64 / 128 / 256 instance, FAST (F % 32 == 0, aligned) and not, split counts 1..32
# with a last split shorter than the others, chunk counts per split that are not a multiple of pj_depth<N>() = 3 / 2 / 1
PJ_CASES = [
    (1, 32, 1, 1),            # one row, one chunk
    (300, 96, 20, 1),         # ragged row tile, fewer than 4 chunks per split
    (130, 640, 64, 5),        # two tiles, 4 chunks per split (not a multiple of 3)
    (257, 4096, 64, 32),      # three tiles, 32 splits of 4 chunks
    (384, 3232, 64, 21),      # 101 chunks: 20 splits of 5 and a last one of 1; tile 2 rotates by 3 of 5 chunks
    (150, 1000, 64, 8),       # F % 32 != 0 (F % 4 == 0): non-FAST vector loads, N = 64
    (128, 4064, 65, 26),      # N = 128: 127 chunks -> 25 splits of 5, the last of 2
    (300, 1600, 100, 10),     # N = 128, 5 chunks per split (not a multiple of 2), tile 2 rotates by 2
    (200, 1000, 128, 8),      # non-FAST vector loads, N = 128
    (700, 1536, 128, 12),
    (129, 4096, 129, 32),     # N = 256, tile 1 rotates by 2
    (64, 130, 256, 1),        # F % 4 != 0: scalar loads, N = 256
]


def _pj_case_check(n_out, F, d, want_splits):
    n_splits, cps, last = pj_splits(n_out, F, d)
    assert n_splits == want_splits, f"pj_plan gives {n_splits} splits (chunks {cps}, last {last}), case claims {want_splits}"
    return n_splits, cps, last


def _pj_operands(rng, n_table, F, d, low_on):
    """(table ints, W ints, table scale, W scale): the side named by `low_on` carries 12-13 significant bits (nonzero
    tf32 lo), the other at most 2 bits, sparse enough for the 2^22 budget."""
    dens = min(1.0, 300.0 / F)
    if low_on == "table":
        T = O.exact_ints(rng, (n_table, F), rng.integers(12, 14), full=True)
        Wt = O.exact_ints(rng, (d, F), 1, density=dens)
    else:
        T = O.exact_ints(rng, (n_table, F), 1, density=dens)
        Wt = O.exact_ints(rng, (d, F), rng.integers(12, 14), full=True)
    return T, Wt


def _pj_bias(rng, d):
    return O.exact_ints(rng, (d,), 12)


@pytest.mark.parametrize("low_on", ["table", "weight"])
@pytest.mark.parametrize("n_out,F,d,splits", PJ_CASES)
def test_project_tc_exact(dev, n_out, F, d, splits, low_on):
    from mmrec_b200 import ops
    _pj_case_check(n_out, F, d, splits)
    rng = np.random.default_rng(n_out + F + d)
    n_table = n_out + 37
    T, Wt = _pj_operands(rng, n_table, F, d, low_on)
    idx = rng.integers(0, n_table, n_out)                            # unsorted, duplicated
    idx[-1] = n_table - 1                                            # the last row of the table
    ts, ws = 2.0 ** -13, 2.0 ** -3
    O.assert_exact_matmul(T[idx], Wt.T)
    b = _pj_bias(rng, d)
    exact = O.int_matmul(T[idx], Wt.T)
    with_b = exact + b[None, :]
    assert int(np.abs(with_b).max()) < (1 << 24)
    table = torch.from_numpy(O.to_f32_exact(T, ts)).to(dev)
    W = torch.from_numpy(O.to_f32_exact(Wt, ws)).to(dev)
    bias = torch.from_numpy(O.to_f32_exact(b, ts * ws)).to(dev)
    ops.set_project_path(True)
    got = ops.project_raw(table, W, bias, torch.from_numpy(idx).to(dev))
    O.assert_bits(got, O.to_f32_exact(with_b, ts * ws), f"gathered + bias ({low_on} carries the low bits)")
    got = ops.project_raw(table[:n_out], W, None)
    O.assert_bits(got, O.to_f32_exact(O.int_matmul(T[:n_out], Wt.T), ts * ws), f"whole table, no bias ({low_on} carries the low bits)")


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("n_out,F,d", [(300, 512, 64), (200, 100, 20), (130, 1028, 128), (90, 256, 256), (50, 96, 300)])
def test_project_l2_normalize_and_misaligned_table(dev, n_out, F, d, path):
    """The row L2 norm (`1 / max(sqrt(ss), 1e-12)`, emulated: ss is an exact integer) on both paths, d > 256 on the SIMT
    path's generic kernel, and a table 4 bytes off 16-byte alignment (non-vector loads on the tensor-core path)."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(F + d)
    T = O.exact_ints(rng, (n_out, F), 2)
    Wt = O.exact_ints(rng, (d, F), 1, density=min(1.0, 8.0 / F * 8))
    Y = O.int_matmul(T, Wt.T)
    O.assert_exact_matmul(T, Wt.T)
    assert int((Y * Y).sum(1).max()) < O.EXACT_BUDGET
    b = O.exact_ints(rng, (d,), 2)
    Yb = Y + b
    assert int((Yb * Yb).sum(1).max()) < O.EXACT_BUDGET
    buf = torch.empty(n_out * F + 4, device=dev)
    table = buf[1:1 + n_out * F].view(n_out, F)
    table.copy_(torch.from_numpy(O.to_f32_exact(T, 1.0)))
    assert table.data_ptr() % 16 != 0 and table.is_contiguous()
    W = torch.from_numpy(O.to_f32_exact(Wt, 1.0)).to(dev)
    ops.set_project_path(path == "tc")
    try:
        got = ops.project_raw(table, W, torch.from_numpy(O.to_f32_exact(b, 1.0)).to(dev), l2_normalize=True)
        O.assert_bits(got, O.l2_rows_f32(O.to_f32_exact(Yb, 1.0)), f"{path}: l2-normalised rows")
        got = ops.project_raw(table, W, None)
        O.assert_bits(got, O.to_f32_exact(Y, 1.0), f"{path}: misaligned table")
    finally:
        ops.set_project_path(True)


# ======================================================================================================================
# K3t: unfused scoring (+ mask + top-k)
# ======================================================================================================================
@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("low_on", ["user", "item"])
@pytest.mark.parametrize("B,I,d", [(130, 300, 40), (257, 513, 48), (1, 1000, 96), (300, 257, 96)])
def test_score_exact(dev, B, I, d, low_on, path):
    from mmrec_b200 import ops
    rng = np.random.default_rng(B + I + d)
    n_users = B + 50
    hi = lambda shape: O.exact_ints(rng, shape, rng.integers(12, 14), full=True)
    lo = lambda shape: O.exact_ints(rng, shape, 2)
    Ui, Ii = (hi((n_users, d)), lo((I, d))) if low_on == "user" else (lo((n_users, d)), hi((I, d)))
    users = rng.integers(0, n_users, B)
    O.assert_exact_matmul(Ui[users], Ii.T)
    want = O.to_f32_exact(O.int_matmul(Ui[users], Ii.T), 2.0 ** -10)
    ue = torch.from_numpy(O.to_f32_exact(Ui, 2.0 ** -9)).to(dev)
    ie = torch.from_numpy(O.to_f32_exact(Ii, 2.0 ** -1)).to(dev)
    ops.set_score_path(path)
    try:
        got = ops.score(ue, ie, torch.from_numpy(users).to(dev))
    finally:
        ops.set_score_path("auto")
    O.assert_bits(got, want, f"{path} scores ({low_on} carries the low bits)")


@pytest.mark.parametrize("path", ["tc", "simt"])
@pytest.mark.parametrize("B,I,d,k", [(70, 3000, 48, 50), (129, 700, 40, 20), (3, 513, 96, 256)])
def test_score_mask_topk_on_integer_scores(dev, B, I, d, k, path):
    """Small integer scores: hundreds of exact ties per row; mask_topk must order them by ascending item index."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(B + I)
    Ui = O.exact_ints(rng, (B, d), 1, density=0.3)
    Ii = O.exact_ints(rng, (I, d), 1, density=0.3)
    mask = np.stack([rng.integers(0, B, 4 * B), rng.integers(0, I, 4 * B)])
    s = O.to_f32_exact(O.int_matmul(Ui, Ii.T), 1.0)
    sm = s.copy()
    sm[mask[0], mask[1]] = O.MASKED_SCORE
    wv, wi = O.topk_tie_low_index(sm, k)
    ops.set_score_path(path)
    try:
        S = ops.score(torch.from_numpy(O.to_f32_exact(Ui, 1.0)).to(dev), torch.from_numpy(O.to_f32_exact(Ii, 1.0)).to(dev))
    finally:
        ops.set_score_path("auto")
    O.assert_bits(S, s, f"{path} integer scores")
    val, idx = ops.mask_topk(S, torch.from_numpy(mask).to(dev), k)
    O.assert_bits(val, wv, "top-k values")
    assert np.array_equal(idx.cpu().numpy(), wi), "top-k indices (ties towards the lower index)"


# ======================================================================================================================
# precision of the 3xTF32 paths on positive full-mantissa operands
# ======================================================================================================================
@pytest.mark.parametrize("kernel,F", [("project", 256), ("project", 4096), ("score", 40), ("score", 128)])
def test_tf32_paths_per_element_bound(dev, kernel, F):
    """Every element within (3 * 2^-20 + (steps + splits + 1) * 2 * 2^-24) * sum |a||b| of the exact value.

    With positive operands sum |a||b| = |result|, so the bound is tight enough to separate 3xTF32 from anything less.
    Per product a*b (a the table / user side, b the weights / items):
      * K2 table, truncating split: hi exact, the tensor core truncates lo to tf32: <= 2^-10 |lo| <= 2^-20 |a|;
      * round-to-nearest split (K2 weights, both K3t operands): |b - hi - lo| <= 2^-11 |b - hi| <= 2^-22 |b|;
      * the dropped lo*lo term: <= 2^-10 |a| * 2^-11 |b| = 2^-21 |ab|;
      so <= (2^-20 + 2^-22 + 2^-21) |ab| < 3 * 2^-20 |ab| per product, summed: 3 * 2^-20 sum |a||b|.
    Accumulation: every wgmma adds into the fp32 accumulator (`steps` = 3 per 8-deep K step of a split), then the K
    splits are added (`splits`) and the bias (1); each is at most one ulp (2 * 2^-24, allowing truncation) of a partial
    sum <= sum |a||b| on positive data.
    A 1xTF32 product, or a missing lo term, errs by ~2^-11 ~ 5e-4 relative on such data on average."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(F)
    if kernel == "project":
        n, d = 300, 64
        a = (rng.random((n, F)) + 0.5).astype(np.float32)
        b = (rng.random((d, F)) + 0.5).astype(np.float32)
        n_splits, cps, _ = pj_splits(n, F, d)
        steps = 3 * cps * 32 // 8
        ops.set_project_path(True)
        got = ops.project_raw(torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev), None).cpu().numpy()
    else:                                                                 # K3t: the contraction depth is d = F <= 128
        a = (rng.random((200, F)) + 0.5).astype(np.float32)
        b = (rng.random((700, F)) + 0.5).astype(np.float32)
        n_splits, steps = 0, 3 * (-(-F // 32) * 32) // 8
        ops.set_score_path("tc")
        try:
            got = ops.score(torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)).cpu().numpy()
        finally:
            ops.set_score_path("auto")
    exact = a.astype(np.float64) @ b.astype(np.float64).T                 # = sum |a||b| (positive operands)
    bound = (3 * 2.0 ** -20 + (steps + n_splits + 1) * 2 * 2.0 ** -24) * exact
    err = np.abs(got.astype(np.float64) - exact)
    worst = float((err / exact).max())
    assert (err <= bound).all(), f"{kernel} F={F}: worst relative error {worst:.3e} over the bound {float((bound / exact).max()):.3e}"


# ======================================================================================================================
# K5: training kernels
# ======================================================================================================================
@pytest.mark.parametrize("n_idx,n_rows,d", [(0, 10, 64), (1, 1, 1), (4096, 7000, 64), (20000, 300, 100), (9000, 70, 256), (500, 100000, 32),
                                            (700, 333, 300)])
def test_index_sum_rows_exact(dev, n_idx, n_rows, d):
    from mmrec_b200 import ops
    rng = np.random.default_rng(n_idx + d)
    idx = rng.integers(0, n_rows, n_idx)
    g = O.exact_ints(rng, (n_idx, d), 6)
    want = np.zeros((n_rows, d), np.int64)
    np.add.at(want, idx, g)
    cnt = np.bincount(idx, minlength=n_rows) if n_idx else np.zeros(n_rows, np.int64)
    assert int(cnt.max(initial=0)) * 63 < O.EXACT_BUDGET
    got = ops.index_sum_rows(torch.from_numpy(O.to_f32_exact(g, 2.0 ** -5)).reshape(n_idx, d).to(dev), torch.from_numpy(idx).to(dev), n_rows)
    O.assert_bits(got, O.to_f32_exact(want, 2.0 ** -5), "index_sum_rows")


@pytest.mark.parametrize("n,n_table,F,d,gather,bias", [
    (7000, 7000, 4096, 64, False, True),
    (4096, 7000, 4096, 64, True, True),
    (7000, 7000, 384, 64, False, True),
    (1000, 1000, 516, 128, False, False),
    (37, 50, 100, 20, True, True),
    (333, 333, 130, 64, False, True),
    (50, 64, 77, 300, True, True),
    (1, 1, 4, 1, False, True),
])
def test_linear_wgrad_exact(dev, n, n_table, F, d, gather, bias):
    from mmrec_b200 import ops
    rng = np.random.default_rng(n + F + d)
    T = O.exact_ints(rng, (n_table, F), 3)
    up = O.exact_ints(rng, (n, d), 3, density=min(1.0, 2000.0 / n))
    idx = rng.integers(0, n_table, n) if gather else None
    x = T if idx is None else T[idx]
    O.assert_exact_matmul(up.T, x)
    dW, db = ops.linear_wgrad(torch.from_numpy(O.to_f32_exact(up, 2.0 ** -4)).to(dev), torch.from_numpy(O.to_f32_exact(T, 0.5)).to(dev),
                              None if idx is None else torch.from_numpy(idx).to(dev), want_bias=bias)
    O.assert_bits(dW, O.to_f32_exact(O.int_matmul(up.T, x), 2.0 ** -5), "dW")
    if bias:
        O.assert_bits(db, O.to_f32_exact(up.sum(0), 2.0 ** -4), "db")


# DgradShape<64, 512> (d <= 64) and <128, 256> (d > 64, k chunks of 128 accumulated by the store form); STORE (aligned,
# F % 4 == 0, d <= 128) and STORE_ANY (F % 4 != 0, or d > 128)
@pytest.mark.parametrize("n_rows,F,d", [(7000, 4096, 64), (7000, 384, 64), (333, 1028, 128), (17, 8, 3), (1, 4, 1), (5000, 512, 96),
                                        (333, 130, 64), (129, 200, 256), (50, 77, 300), (600, 1030, 100), (300, 516, 65)])
def test_linear_dgrad_exact(dev, n_rows, F, d):
    from mmrec_b200 import ops
    rng = np.random.default_rng(n_rows + F + d)
    G = O.exact_ints(rng, (n_rows, d), 8)
    W = O.exact_ints(rng, (d, F), 4)
    O.assert_exact_matmul(G, W)
    got = ops.linear_dgrad(torch.from_numpy(O.to_f32_exact(G, 2.0 ** -8)).to(dev), torch.from_numpy(O.to_f32_exact(W, 2.0 ** -2)).to(dev))
    O.assert_bits(got, O.to_f32_exact(O.int_matmul(G, W), 2.0 ** -10), "G @ W")


# ======================================================================================================================
# Adam
# ======================================================================================================================
LR, B1, B2, EPS = 1e-3, 0.9, 0.999, 1e-8


def _torch_foreach_adam(dev, p0, grads, wd):
    p = torch.nn.Parameter(torch.as_tensor(p0).to(dev).clone())
    opt = torch.optim.Adam([p], lr=LR, betas=(B1, B2), eps=EPS, weight_decay=wd, foreach=True)
    for g in grads:
        p.grad = torch.as_tensor(g).to(dev).clone()
        opt.step()
    st = opt.state[p]
    return p.detach(), st["exp_avg"], st["exp_avg_sq"]


def _emulate(p0, grads, wd):
    p, m, v = np.asarray(p0, np.float32), np.zeros_like(p0, np.float32), np.zeros_like(p0, np.float32)
    for t, g in enumerate(grads, 1):
        p, m, v = O.adam_foreach_f32(p, g, m, v, t, LR, B1, B2, EPS, wd)
    return p, m, v


def _assert_adam(got, want, what):
    (p, m, v), (wp, wm, wv) = ((x.detach().cpu() if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x, np.float32))
                                for x in t) for t in (got, want))
    diff = float((v != wv).double().mean())
    O.assert_bits(m, wm, f"{what}: exp_avg")
    assert diff == 0.0, f"{what}: {100 * diff:.2f} % of exp_avg_sq elements differ"
    O.assert_bits(v, wv, f"{what}: exp_avg_sq")
    O.assert_bits(p, wp, f"{what}: param")


@pytest.mark.parametrize("wd", [0.0, 0.05])
def test_adam_foreach_emulation_equals_torch(dev, wd):
    rng = np.random.default_rng(3)
    p0 = rng.standard_normal(100003).astype(np.float32)
    grads = [(0.05 * rng.standard_normal(p0.shape)).astype(np.float32) for _ in range(3)]
    _assert_adam(_emulate(p0, grads, wd), _torch_foreach_adam(dev, p0, grads, wd), "oracle.adam_foreach_f32 vs torch")


@pytest.mark.parametrize("wd", [0.0, 0.05])
def test_adam_step_bitwise_equals_torch(dev, wd):
    """`mmrec_adam_f32` (vector and scalar paths, > 24 tensors: two launches) against torch.optim.Adam(foreach=True)."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(5)
    shapes = [(20000, 64), (64, 4096), (4097,), (1,), (3, 5, 7)] + [(11,)] * 25
    ps = [rng.standard_normal(s).astype(np.float32) for s in shapes]
    steps = [[(0.05 * rng.standard_normal(s)).astype(np.float32) for s in shapes] for _ in range(3)]
    cur = [torch.from_numpy(p).to(dev) for p in ps]
    buf = torch.zeros(4097 + 1, device=dev)
    cur[2] = buf[1:]; cur[2].copy_(torch.from_numpy(ps[2]))                 # unaligned: the scalar path
    ms, vs = [torch.zeros_like(c) for c in cur], [torch.zeros_like(c) for c in cur]
    for t, grads in enumerate(steps, 1):
        gd = [torch.from_numpy(g).to(dev) for g in grads]
        ops.adam_step([(cur[i], gd[i], ms[i], vs[i], -LR / (1 - B1 ** t), (1 - B2 ** t) ** 0.5) for i in range(len(ps))], B1, B2, EPS, wd)
    for i in (0, 1, 2, 3, 4, 29):
        want = _torch_foreach_adam(dev, ps[i], [st[i] for st in steps], wd)
        _assert_adam((cur[i], ms[i], vs[i]), want, f"adam_step {shapes[i]}")


@pytest.mark.parametrize("wd", [0.0, 0.05])
@pytest.mark.parametrize("n_rows,F,d", [(1500, 384, 64), (300, 260, 128)])
def test_linear_dgrad_adam_bitwise_equals_torch(dev, n_rows, F, d, wd):
    """The fused table step with an exactly representable gradient G @ W against torch's Adam on that gradient."""
    from mmrec_b200 import ops
    rng = np.random.default_rng(n_rows + F)
    p0 = rng.standard_normal((n_rows, F)).astype(np.float32)
    W = O.exact_ints(rng, (d, F), 4)
    Gs = [O.exact_ints(rng, (n_rows, d), 8) for _ in range(3)]
    for G in Gs:
        O.assert_exact_matmul(G, W)
    grads = [O.to_f32_exact(O.int_matmul(G, W), 2.0 ** -16) for G in Gs]
    Wd = torch.from_numpy(O.to_f32_exact(W, 2.0 ** -6)).to(dev)
    p = torch.from_numpy(p0).to(dev)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    for t, G in enumerate(Gs, 1):
        ops.linear_dgrad_adam(torch.from_numpy(O.to_f32_exact(G, 2.0 ** -10)).to(dev), Wd, p, m, v, B1, B2, EPS, wd, -LR / (1 - B1 ** t),
                              (1 - B2 ** t) ** 0.5)
    _assert_adam((p, m, v), _torch_foreach_adam(dev, p0, grads, wd), "linear_dgrad_adam")


@pytest.mark.parametrize("wd", [0.0, 0.05])
def test_fused_adam_bitwise_equals_torch_foreach_adam(dev, wd):
    from mmrec_b200.optim import FusedAdam
    rng = np.random.default_rng(9)
    shapes = [(500, 128), (64, 128), (64,), (7,)]
    init = [rng.standard_normal(s).astype(np.float32) for s in shapes]
    a = [torch.nn.Parameter(torch.from_numpy(x).to(dev)) for x in init]
    b = [torch.nn.Parameter(torch.from_numpy(x).to(dev)) for x in init]
    oa = FusedAdam(a, lr=LR, betas=(B1, B2), eps=EPS, weight_decay=wd, factored=False)
    ob = torch.optim.Adam(b, lr=LR, betas=(B1, B2), eps=EPS, weight_decay=wd, foreach=True)
    for _ in range(3):
        for x, y, s in zip(a, b, shapes):
            g = torch.from_numpy((0.05 * rng.standard_normal(s)).astype(np.float32)).to(dev)
            x.grad, y.grad = g.clone(), g.clone()
        oa.step(); ob.step()
    for x, y, s in zip(a, b, shapes):
        _assert_adam((x.detach(), oa.state[x]["exp_avg"], oa.state[x]["exp_avg_sq"]),
                     (y.detach(), ob.state[y]["exp_avg"], ob.state[y]["exp_avg_sq"]), f"FusedAdam {s}")
