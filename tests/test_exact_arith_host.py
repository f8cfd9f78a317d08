"""The host helpers behind tests/test_gpu_exact_arith.py (no GPU): exact operand generators, the exactness precondition,
the fp32 epilogue emulations and the restatement of torch's foreach Adam step.

Each emulation that claims one rounding is compared with `fractions.Fraction` arithmetic followed by a single
round-to-nearest-even to fp32."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import mmrec_oracle as O


def f32_round(x: Fraction) -> np.float32:
    """Nearest fp32 (ties to even) of an exact rational in the normal range."""
    if x == 0:
        return np.float32(0.0)
    s, a = (-1 if x < 0 else 1), abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if a < Fraction(2) ** e:
        e -= 1
    scaled = a / Fraction(2) ** (e - 23)                          # in [2^23, 2^24)
    q, r = divmod(scaled.numerator, scaled.denominator)
    rem = Fraction(r, scaled.denominator)
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and q % 2 == 1):
        q += 1
    return np.float32(s * q * 2.0 ** (e - 23))


def F(x) -> Fraction:
    return Fraction(float(x))


def test_f32_round_reference_itself():
    rng = np.random.default_rng(0)
    for v in rng.standard_normal(200).astype(np.float32):
        assert f32_round(F(v)) == v
    one = Fraction(1)
    assert f32_round(one + Fraction(1, 2 ** 24)) == np.float32(1.0)                       # tie -> even
    assert f32_round(one + Fraction(3, 2 ** 24)) == np.float32(1.0 + 2.0 ** -22)          # tie -> even (up)
    assert f32_round(one + Fraction(1, 2 ** 24) + Fraction(1, 2 ** 40)) == np.float32(1.0 + 2.0 ** -23)


@pytest.mark.parametrize("bits", [1, 2, 11, 12, 13])
def test_exact_ints_bit_budget(bits):
    rng = np.random.default_rng(bits)
    m = O.exact_ints(rng, (4000,), bits)
    assert int(np.abs(m).max()) < 2 ** bits and (m < 0).any() and (m > 0).any()
    full = O.exact_ints(rng, (4000,), bits, full=True)
    assert (O.significant_bits(full) == bits).all()
    sparse = O.exact_ints(rng, (20000,), bits, density=0.1, full=True)
    assert 0.05 < float((sparse != 0).mean()) < 0.15
    assert O.significant_bits(np.array([0, 1, 6, 5, -12, 2 ** 20])).tolist() == [0, 1, 2, 3, 2, 1]


@pytest.mark.parametrize("scale_exp", [-13, -3, 0, 7])
def test_tf32_splits_of_generated_values_are_exact(scale_exp):
    """12-13 significant bits: both splits leave a nonzero lo that tf32 holds exactly; <= 11 bits: lo = 0."""
    rng = np.random.default_rng(scale_exp + 50)
    for bits in (12, 13):
        x = O.to_f32_exact(O.exact_ints(rng, (5000,), bits, full=True), 2.0 ** scale_exp)
        hi, lo, lo_tc = O.tf32_split_trunc(x)
        assert np.array_equal(hi.astype(np.float64) + lo, x.astype(np.float64)) and np.array_equal(lo, lo_tc) and (lo != 0).all()
        hi, lo = O.tf32_split_rn(x)
        assert np.array_equal(hi.astype(np.float64) + lo, x.astype(np.float64)) and (lo != 0).all()
        assert np.array_equal(O.tf32_split_rn(lo)[0], lo)                          # lo is a tf32 value
    x = O.to_f32_exact(O.exact_ints(rng, (5000,), 11), 2.0 ** scale_exp)
    assert (O.tf32_split_trunc(x)[1] == 0).all() and (O.tf32_split_rn(x)[1] == 0).all()


def test_tf32_rn_split_rounds_to_nearest_ties_away():
    x = np.array([1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, -(1 + 2.0 ** -11), 1 + 2.0 ** -11 + 2.0 ** -20], np.float32)
    hi, lo = O.tf32_split_rn(x)
    assert hi.tolist() == [1 + 2.0 ** -10, 1 + 2 * 2.0 ** -10, -(1 + 2.0 ** -10), 1 + 2.0 ** -10]
    assert np.array_equal(hi.astype(np.float64) + lo, x.astype(np.float64))
    # truncation: 1 + 2^-11 keeps hi = 1
    assert O.tf32_split_trunc(x[:1])[0].tolist() == [1.0]


def test_precondition_holds_and_is_detected_when_broken():
    rng = np.random.default_rng(1)
    a = O.exact_ints(rng, (50, 300), 12, full=True)
    b = O.exact_ints(rng, (300, 40), 1, density=0.5)
    s = O.exact_matmul_bound(a, b)
    assert s == int((np.abs(a) @ np.abs(b)).max())
    O.assert_exact_matmul(a, b)
    with pytest.raises(AssertionError, match="precondition"):
        O.assert_exact_matmul(a, np.full_like(b, 7))                                # dense, larger: over 2^22
    with pytest.raises(AssertionError, match="not exact"):
        O.exact_matmul_bound(np.array([[2 ** 13]]), np.array([[2 ** 11]]))          # one product needs 25 bits
    with pytest.raises(AssertionError):
        O.to_f32_exact(np.array([2 ** 24 + 1]), 1.0)
    with pytest.raises(AssertionError):
        O.to_f32_exact(np.array([3]), 0.3)
    assert O.to_f32_exact(np.array([2 ** 24 - 1]), 2.0 ** -30)[0] == (2 ** 24 - 1) * 2.0 ** -30


def test_fdiv_and_epilogue_are_single_roundings():
    rng = np.random.default_rng(2)
    y = O.to_f32_exact(O.exact_ints(rng, (40, 8), 12), 2.0 ** -4)
    acc_in = O.to_f32_exact(O.exact_ints(rng, (40, 8), 12), 2.0 ** -4)
    post = O.to_f32_exact(O.exact_ints(rng, (40, 8), 6), 2.0 ** -9)
    for div in (3.0, 4.0, 7.0):
        Y, acc = O.spmm_epilogue_f32(y, acc_in, div, post=post)
        assert np.array_equal(Y, y)
        for i in range(40):
            for j in range(8):
                q = f32_round((F(y[i, j]) + F(acc_in[i, j])) / F(div))             # y + acc_in is exact: one rounding
                assert O.fdiv_f32(y[i, j] + acc_in[i, j], div) == q
                assert acc[i, j] == f32_round(F(q) + F(post[i, j]))
    Y, acc = O.spmm_epilogue_f32(y, acc_in, 1.0, y_old=acc_in)
    assert np.array_equal(Y, acc) and np.array_equal(acc.astype(np.float64), y.astype(np.float64) + acc_in)


def _sqrt_f32_ok(x, r):
    """r is the correctly rounded fp32 square root of the fp32 x."""
    up, dn = np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(0))
    lo_mid, hi_mid = (F(r) + F(dn)) / 2, (F(r) + F(up)) / 2
    return lo_mid ** 2 <= F(x) <= hi_mid ** 2


def test_gate_and_l2_emulations_step_by_step():
    """Each step of the cosine gate and of the row L2 norm is one IEEE rounding of exact inputs."""
    rng = np.random.default_rng(3)
    y = O.to_f32_exact(O.exact_ints(rng, (30, 256), 7), 1.0)                         # |y|, |ref| < 2^7 at d = 256: sums exact
    ref = O.to_f32_exact(O.exact_ints(rng, (30, 256), 7), 1.0)
    y[0] = 0.0
    Yg, _ = O.spmm_epilogue_f32(y, None, 1.0, gate_ref=ref)
    for i in range(30):
        dot = sum(F(a) * F(b) for a, b in zip(y[i], ref[i]))
        ny, nr = sum(F(a) ** 2 for a in y[i]), sum(F(b) ** 2 for b in ref[i])
        assert max(abs(dot), ny, nr) < 2 ** 24                                      # exact in fp32
        sy, sr = np.sqrt(np.float32(ny)), np.sqrt(np.float32(nr))
        assert _sqrt_f32_ok(np.float32(ny), sy) and _sqrt_f32_ok(np.float32(nr), sr)
        den = f32_round(F(max(sy, np.float32(1e-8))) * F(max(sr, np.float32(1e-8))))
        c = f32_round(dot / F(den))
        want = np.array([f32_round(F(v) * F(c)) for v in y[i]], np.float32)
        assert np.array_equal(Yg[i], want), i
    assert (Yg[0] == 0).all()
    yl = y[:, :64] / np.float32(8.0)
    got = O.l2_rows_f32(yl)
    for i in range(30):
        ss = sum(F(v) ** 2 for v in yl[i])
        s = np.sqrt(np.float32(ss))
        assert F(np.float32(ss)) == ss and _sqrt_f32_ok(np.float32(ss), s)
        inv = f32_round(Fraction(1) / F(max(s, np.float32(1e-12))))
        assert np.array_equal(got[i], np.array([f32_round(F(v) * F(inv)) for v in yl[i]], np.float32)), i


def test_adam_foreach_f32_follows_the_foreach_roundings():
    """One step from zero state, element by element, against exact rational arithmetic with one rounding per op."""
    rng = np.random.default_rng(4)
    p = rng.standard_normal(300).astype(np.float32)
    g = (0.05 * rng.standard_normal(300)).astype(np.float32)
    m0 = (0.01 * rng.standard_normal(300)).astype(np.float32)
    v0 = (1e-4 * rng.random(300)).astype(np.float32)
    lr, b1, b2, eps, wd, step = 1e-3, 0.9, 0.999, 1e-8, 0.05, 3
    P, M, V = O.adam_foreach_f32(p, g, m0, v0, step, lr, b1, b2, eps, wd)
    f = np.float32
    step_size, bc2s = f((lr / (1 - b1 ** step)) * -1), f((1 - b2 ** step) ** 0.5)
    for i in range(300):
        gr = f32_round(F(f(wd)) * F(p[i]) + F(g[i]))
        m = f32_round(F(f(1 - b1)) * F(f32_round(F(gr) - F(m0[i]))) + F(m0[i]))
        v = f32_round(F(f(1 - b2)) * F(f32_round(F(gr) ** 2)) + F(f32_round(F(v0[i]) * F(f(b2)))))
        s = np.sqrt(np.float32(v))
        assert _sqrt_f32_ok(np.float32(v), s)
        den = f32_round(F(f32_round(F(s) / F(bc2s))) + F(f(eps)))
        pn = f32_round(F(step_size) * F(f32_round(F(m) / F(den))) + F(p[i]))
        assert (M[i], V[i], P[i]) == (m, v, pn), i


def test_adam_second_moment_forms_differ_by_one_ulp():
    """The form torch computes, fma(1 - beta2, g * g, v * beta2), and fma((1 - beta2) * g, g, v * beta2) round
    differently (by one or two ulps) on a large share of elements after the first step (v = 0), and on fewer later."""
    rng = np.random.default_rng(5)
    g = (0.05 * rng.standard_normal(200000)).astype(np.float32)
    w2, b2 = np.float32(1 - 0.999), np.float32(0.999)
    v_new = O.fmaf32(w2, (g * g).astype(np.float32), np.float32(0.0))
    v_old = O.fmaf32((w2 * g).astype(np.float32), g, np.float32(0.0))
    first = float((v_new != v_old).mean())
    assert 0.2 < first < 0.5, first
    ulps = np.abs(v_new.view(np.int32).astype(np.int64) - v_old.view(np.int32))
    assert int(ulps.max()) <= 2                                                      # two roundings each
    g2 = (0.05 * rng.standard_normal(200000)).astype(np.float32)
    vb = (v_new * b2).astype(np.float32)
    later = float((O.fmaf32(w2, (g2 * g2).astype(np.float32), vb) != O.fmaf32((w2 * g2).astype(np.float32), g2, vb)).mean())
    assert 0.0 < later < first, later
    assert math.isfinite(first)


def test_assert_bits_reports_the_first_difference_and_matches_nans():
    a = np.array([[1.0, np.nan], [3.0, 4.0]], np.float32)
    O.assert_bits(a, a.copy(), "same")
    b = a.copy()
    b[1, 0] = np.nextafter(np.float32(3.0), np.float32(4.0))
    with pytest.raises(AssertionError, match=r"1 of 4 elements differ; first at \(1, 0\)"):
        O.assert_bits(b, a, "one ulp")
    c = a.copy()
    c[0, 0] = np.nan
    with pytest.raises(AssertionError, match="1 of 4"):
        O.assert_bits(c, a, "NaN against a number")


@pytest.mark.parametrize("with_bias", [True, False])
def test_fuse_chain_is_a_sequential_fmaf_chain(with_bias):
    """acc = b (or +0), then acc = fl(W[j, k] x_k + acc) for k = 0 .. d-1, each step one rounding of the exact value."""
    rng = np.random.default_rng(6)
    n, d = 5, 32
    W = rng.standard_normal((d, d)).astype(np.float32)
    X = (rng.standard_normal((n, d)) * np.exp2(rng.integers(-20, 20, (n, d)))).astype(np.float32)   # cancellation, mixed scales
    X[1] = 0.0
    b = rng.standard_normal(d).astype(np.float32) if with_bias else None
    got = O.fuse_chain_f32(X, W, b)
    for i in range(n):
        for j in range(d):
            acc = np.float32(0.0) if b is None else b[j]
            for k in range(d):
                acc = f32_round(F(W[j, k]) * F(X[i, k]) + F(acc))
            assert got[i, j] == acc, (i, j)
    assert np.array_equal(got[1], np.zeros(d, np.float32) if b is None else b)


def test_csr_coalesce_sums_each_run_in_input_order():
    """A stable sort by row * n_cols + col, then a sequential fp32 sum per key in input order; without summing, equal
    keys keep their input order and their values."""
    rng = np.random.default_rng(7)
    n_rows, n_cols, nnz = 6, 5, 400
    row, col = rng.integers(1, n_rows - 1, nnz), rng.integers(0, n_cols, nnz)      # rows 0 and 5 empty
    val = (rng.standard_normal(nnz) * np.exp2(rng.integers(-12, 12, nnz))).astype(np.float32)
    rowptr, colidx, vals = O.csr_coalesce_f32(row, col, val, n_rows, n_cols)
    order = sorted(range(nnz), key=lambda i: (row[i], col[i]))                      # Python's sort is stable
    keys, sums = [], []
    for i in order:
        if keys and keys[-1] == (row[i], col[i]):
            sums[-1] = np.float32(sums[-1] + val[i])
        else:
            keys.append((row[i], col[i]))
            sums.append(val[i])
    assert colidx.tolist() == [c for _, c in keys] and np.array_equal(vals, np.array(sums, np.float32))
    assert rowptr.tolist() == [sum(1 for r, _ in keys if r < q) for q in range(n_rows + 1)]
    backwards = [np.float32(0)] * len(keys)                                          # the order is visible in the bits
    for i in reversed(order):
        k = keys.index((row[i], col[i]))
        backwards[k] = np.float32(backwards[k] + val[i])
    assert not np.array_equal(vals, np.array(backwards, np.float32))
    _, c1, v1 = O.csr_coalesce_f32(row, col, None, n_rows, n_cols)                   # no values: each entry counts 1
    assert np.array_equal(v1, np.array([sum(1 for i in order if (row[i], col[i]) == kk) for kk in keys], np.float32))
    rp, c2, v2 = O.csr_coalesce_f32(row, col, val, n_rows, n_cols, sum_duplicates=False)
    assert c2.tolist() == [col[i] for i in order] and np.array_equal(v2, val[order]) and rp[-1] == nnz
    rp, c0, v0 = O.csr_coalesce_f32(np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32), 3, 4)
    assert rp.tolist() == [0, 0, 0, 0] and c0.size == 0 and v0.size == 0


def test_bipartite_norm_is_four_ieee_operations_per_side():
    eps = 1e-7
    users = np.array([0, 0, 1, 3, 3, 3], np.int64)
    items = np.array([1, 0, 1, 1, 2, 1], np.int64)
    got = O.bipartite_norm_f32(users, items, 5, 4, eps)

    def side(deg):
        x = f32_round(F(np.float32(deg)) + F(np.float32(eps)))
        s = np.sqrt(np.float32(x))
        assert _sqrt_f32_ok(np.float32(x), s)
        return f32_round(Fraction(1) / F(s))

    du, di = np.bincount(users, minlength=5), np.bincount(items, minlength=4)
    for e in range(users.size):
        assert got[e] == f32_round(F(side(du[users[e]])) * F(side(di[items[e]]))), e
    # the degree's int -> float conversion rounds to nearest even above 2^24
    big = O.bipartite_norm_f32(np.zeros((1 << 24) + 3, np.int64), np.arange((1 << 24) + 3) % 3, 1, 3)
    assert big[0] == f32_round(F(side((1 << 24) + 4)) * F(side(-(-((1 << 24) + 3) // 3))))          # item 0: ceil(n / 3) edges
