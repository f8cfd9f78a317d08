"""The host emulation of the fused scorer's fp32 arithmetic (oracle/mmrec_oracle.py: fmaf32, cf_chain_scores,
topk_float_key, cf_exact_topk) against exact rational arithmetic and straightforward scalar restatements.  No GPU:
tests/test_gpu_score_exact.py holds the kernels to these functions bit for bit, so they must be right first."""
import math
from fractions import Fraction

import numpy as np
import torch

from oracle import mmrec_oracle as O

F32_MAX = float(np.finfo(np.float32).max)


def f32_bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def round_f32(x: Fraction, zero_sign: float = 1.0) -> np.float32:
    """Correct rounding of an exact rational to float32 (nearest, ties to even, subnormals, overflow to inf)."""
    if x == 0:
        return np.float32(math.copysign(0.0, zero_sign))
    ax = abs(x)
    e = ax.numerator.bit_length() - ax.denominator.bit_length()      # 2^e <= ax < 2^(e+2)
    if Fraction(2) ** e > ax:
        e -= 1
    if Fraction(2) ** (e + 1) <= ax:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    q = ax / ulp
    n = q.numerator // q.denominator
    rem = q - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    val = n * ulp
    if val >= Fraction(2) ** 128:
        out = math.inf
    else:
        out = float(val)                                              # exact: n has at most 24 bits
    return np.float32(out if x > 0 else -out)


def fma_exact(a, b, c) -> np.float32:
    a, b, c = float(a), float(b), float(c)
    if not (math.isfinite(a) and math.isfinite(b) and math.isfinite(c)):
        with np.errstate(all="ignore"):
            r = np.float32(np.float64(a) * np.float64(b) + np.float64(c))
        return np.uint32(0x7FFFFFFF).view(np.float32) if np.isnan(r) else r
    exact = Fraction(a) * Fraction(b) + Fraction(c)
    p_zero_sign = math.copysign(1.0, a) * math.copysign(1.0, b)
    # an exact zero sum: -0 only when both addends are -0 (round to nearest)
    zs = -1.0 if (exact == 0 and a * b == 0 and p_zero_sign < 0 and math.copysign(1.0, c) < 0 and c == 0) else 1.0
    return round_f32(exact, zs)


def check_fma(a, b, c):
    a, b, c = (np.asarray(x, np.float32) for x in (a, b, c))
    got = O.fmaf32(a, b, c)
    want = np.array([fma_exact(x, y, z) for x, y, z in zip(a, b, c)], np.float32)
    bad = np.nonzero(f32_bits(got) != f32_bits(want))[0]
    assert bad.size == 0, f"{bad.size} mismatches, first: fmaf({a[bad[0]]!r}, {b[bad[0]]!r}, {c[bad[0]]!r}) = {got[bad[0]]!r}, want {want[bad[0]]!r}"


def rand_f32(rng, n, lo, hi):
    m = rng.uniform(1.0, 2.0, n)
    e = rng.integers(lo, hi, n)
    s = rng.choice([-1.0, 1.0], n)
    return (s * np.ldexp(m, e)).astype(np.float32)


def test_fmaf32_random_triples():
    rng = np.random.default_rng(0)
    n = 6000
    check_fma(rand_f32(rng, n, -30, 30), rand_f32(rng, n, -30, 30), rand_f32(rng, n, -40, 40))
    # addends of similar size: cancellation
    a, b = rand_f32(rng, n, -3, 3), rand_f32(rng, n, -3, 3)
    check_fma(a, b, (-(a.astype(np.float64) * b) * (1 + rng.uniform(-1e-6, 1e-6, n))).astype(np.float32))


def test_fmaf32_midpoints():
    """s = a*b + c rounded to float64 lands exactly on a float32 midpoint while the exact value is off it by far less
    than a float64 ulp: plain float64 -> float32 conversion gets half of these wrong (double rounding)."""
    rng = np.random.default_rng(1)
    a_l, b_l, c_l = [], [], []
    for _ in range(3000):
        c = float(rand_f32(rng, 1, -20, 20)[0])
        if rng.random() < 0.05:
            c = math.copysign(F32_MAX, c)
        h = 2.0 ** (math.frexp(c)[1] - 25)                           # half an ulp of c
        i, j = int(rng.integers(1, 4)), int(rng.integers(1, 4))
        x, y = 1 + i * 2.0 ** -23, 1 - j * 2.0 ** -23                 # x*y = 1 + (i - j) 2^-23 - i j 2^-46
        if rng.random() < 0.5:
            x, y = 1 - i * 2.0 ** -24, 1 + j * 2.0 ** -23
        sgn = float(rng.choice([-1.0, 1.0]))
        a_l.append(sgn * h * x); b_l.append(y); c_l.append(c)
    a, b, c = np.array(a_l, np.float32), np.array(b_l, np.float32), np.array(c_l, np.float32)
    assert np.array_equal(a.astype(np.float64), np.array(a_l)) and np.array_equal(b.astype(np.float64), np.array(b_l))
    check_fma(a, b, c)
    # the construction really is adversarial: rounding the float64 sum to float32 is wrong for many of these
    with np.errstate(over="ignore"):
        naive = (a.astype(np.float64) * b + c).astype(np.float32)
    assert np.count_nonzero(f32_bits(naive) != f32_bits(O.fmaf32(a, b, c))) > 100


def test_fmaf32_subnormals_zeros_overflow_nonfinite():
    rng = np.random.default_rng(2)
    n = 3000
    # results in and around the subnormal range (products ~2^-150 .. 2^-120, addends ~2^-149 .. 2^-120)
    check_fma(rand_f32(rng, n, -80, -60), rand_f32(rng, n, -80, -60), rand_f32(rng, n, -149, -120))
    sub = np.array([1e-45, -1e-45, 3e-45, 1.1754942e-38, -1.1754942e-38], np.float32)
    check_fma(np.repeat(sub, 5), np.tile(np.array([0.5, -0.5, 2.0, 1.5, -0.75], np.float32), 5), np.tile(sub, 5))
    # signed zeros: every sign combination, and exact cancellation (+0 in round to nearest)
    z = [0.0, -0.0, 1.0, -1.0]
    trip = np.array([(x, y, w) for x in z for y in z for w in [0.0, -0.0, 1.0, -1.0]], np.float32).T
    check_fma(*trip)
    check_fma(np.array([3.0, -3.0, 1e-30], np.float32), np.array([2.0, 2.0, -1e-30], np.float32), np.array([-6.0, 6.0, 0.0], np.float32))
    # overflow: to inf, and just below it
    check_fma(np.array([2.0 ** 64, -2.0 ** 64, 2.0 ** 63, F32_MAX, 1.0], np.float32), np.array([2.0 ** 64, 2.0 ** 64, 2.0 ** 64, 1.0, F32_MAX], np.float32),
              np.array([0.0, 0.0, -F32_MAX, F32_MAX, -F32_MAX], np.float32))
    # non-finite operands: the IEEE result, every NaN as CUDA's canonical +NaN
    inf, nan = np.inf, np.nan
    a = np.array([inf, inf, 0.0, nan, 1.0, -inf, 1.0], np.float32)
    b = np.array([0.0, 1.0, -inf, 1.0, 1.0, 1.0, -nan], np.float32)
    c = np.array([1.0, -inf, 0.0, 0.0, inf, -inf, 0.0], np.float32)
    got = O.fmaf32(a, b, c)
    assert f32_bits(got).tolist() == [0x7FFFFFFF, 0x7FFFFFFF, 0x7FFFFFFF, 0x7FFFFFFF, 0x7F800000, 0xFF800000, 0x7FFFFFFF]


def chain_scalar(u, v):
    """score_cf.cu, "exact fp32 score of one (user, item) pair", one pair, one operation at a time."""
    d = len(u)
    L = 8 if d <= 32 else (16 if d <= 64 else 32)
    uu = [np.float32(x) for x in u] + [np.float32(0)] * (4 * L - d)
    vv = [np.float32(x) for x in v] + [np.float32(0)] * (4 * L - d)
    p = []
    for blk in range(L):
        acc = np.float32(0.0)
        for j in range(4 * blk, 4 * blk + 4):
            acc = fma_exact(uu[j], vv[j], acc)
        p.append(acc)
    w = L // 2
    while w >= 1:
        for a in range(w):
            with np.errstate(all="ignore"):
                p[a] = np.float32(p[a] + p[a + w])
        w //= 2
    r = np.float32(p[0])
    return np.uint32(0x7FFFFFFF).view(np.float32) if np.isnan(r) else r


def test_cf_chain_scores_against_scalar_loop():
    rng = np.random.default_rng(3)
    for d in [1, 3, 4, 5, 31, 32, 33, 63, 64, 65, 100, 127, 128]:
        u = rng.standard_normal((6, d)).astype(np.float32)
        v = rng.standard_normal((6, d)).astype(np.float32)
        u[1] = np.ldexp(u[1], -75); v[1] = np.ldexp(v[1], -70)        # subnormal products and partial sums
        u[2, ::2] = 0.0; v[2] = -np.abs(v[2]); u[2, 1::2] *= -1e-30  # -0 products / partial sums: the padding turns -0 into +0
        u[3] = np.round(u[3] * 8) / 64; v[3] = np.round(v[3] * 8) / 64   # exact arithmetic
        u[4] *= 1e18; v[4] *= 1e19                                    # overflow to inf
        u[5, 0] = np.inf
        got = O.cf_chain_scores(u, v)
        want = np.array([chain_scalar(u[i], v[i]) for i in range(6)], np.float32)
        assert np.array_equal(f32_bits(got), f32_bits(want)), f"d={d}: {got} vs {want}"
    # the zero-padding is part of the arithmetic: a chain ending in -0 comes out +0 once padded blocks are added
    u = np.array([[-1e-30]], np.float32); v = np.array([[1e-30]], np.float32)
    assert f32_bits(O.fmaf32(u[0], v[0], 0.0)) == 0x80000000 and f32_bits(O.cf_chain_scores(u, v)) == 0
    # broadcasting: a row against a table equals the paired form
    u = rng.standard_normal((3, 1, 40)).astype(np.float32); v = rng.standard_normal((1, 50, 40)).astype(np.float32)
    full = O.cf_chain_scores(u, v)
    paired = O.cf_chain_scores(np.broadcast_to(u, (3, 50, 40)).reshape(-1, 40), np.broadcast_to(v, (3, 50, 40)).reshape(-1, 40))
    assert np.array_equal(f32_bits(full).ravel(), f32_bits(paired))


def test_topk_float_key_order():
    nan = np.uint32(0x7FFFFFFF).view(np.float32)
    vals = np.array([[0.0, -0.0, 1.0, nan, 1.0, -np.inf, np.inf, -1e10]], np.float32)
    v, i = O.topk_float_key(vals, 8)
    assert i.tolist() == [[3, 6, 2, 4, 0, 1, 7, 5]]
    assert f32_bits(v[0, 4]) == 0 and f32_bits(v[0, 5]) == 0x80000000
    keys = O.float_key(np.array([-np.inf, -1.0, -0.0, 0.0, 1e-45, 1.0, np.inf, nan], np.float32))
    assert np.all(np.diff(keys.astype(np.int64)) > 0)


def brute_force(ue, ie, users, mask, k, item_offset=0):
    u = ue[users].numpy() if users is not None else ue.numpy()
    s = O.cf_chain_scores(u[:, None, :], ie.numpy()[None, :, :])
    if mask is not None:
        r, c = mask[0].numpy(), mask[1].numpy() - item_offset
        ok = (r >= 0) & (r < s.shape[0]) & (c >= 0) & (c < s.shape[1])
        s[r[ok], c[ok]] = O.MASKED_SCORE
    v, i = O.topk_float_key(s, k)
    return torch.from_numpy(v), torch.from_numpy(i + item_offset)


def test_cf_exact_topk_equals_brute_force():
    """The candidate selection of cf_exact_topk never changes the answer: same bits as emulating every pair."""
    g = torch.Generator().manual_seed(4)
    for (B, U, I, d, k, quant) in [(40, 50, 300, 33, 10, False), (24, 30, 257, 16, 20, True), (9, 9, 130, 128, 50, False)]:
        ue = torch.randn(U, d, generator=g) * 0.1; ie = torch.randn(I, d, generator=g) * 0.1
        if quant:                                                    # multiples of 2^-6: exact scores, many ties
            ue = torch.randint(-3, 4, (U, d), generator=g).float() / 64; ie = torch.randint(-3, 4, (I, d), generator=g).float() / 64
        users = torch.randperm(U, generator=g)[:B]
        off = 1000
        rows = torch.cat([torch.randint(-2, B + 2, (B * 4,), generator=g), torch.full((I - k + 3,), 1)])
        cols = torch.cat([torch.randint(off - 20, off + I + 20, (B * 4,), generator=g), torch.randperm(I, generator=g)[:I - k + 3] + off])
        mask = torch.stack([rows, cols])
        mask = torch.cat([mask, mask[:, :10]], 1)                     # duplicates
        ue[users[2]] = 0.0                                           # a zero row: every item ties at +0
        ue[users[3], 1] = float("inf")                               # a non-finite row
        got_v, got_i = O.cf_exact_topk(ue, ie, users, mask, k, item_offset=off)
        want_v, want_i = brute_force(ue, ie, users, mask, k, item_offset=off)
        assert torch.equal(got_i, want_i)
        assert torch.equal(got_v.view(torch.int32), want_v.view(torch.int32))
        assert torch.all(got_v[1, k - 3:] == O.MASKED_SCORE)         # fewer than k unmasked items: masked ones fill in
        assert torch.all(got_v[2] == 0)
