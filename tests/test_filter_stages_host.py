"""The host restatements of tests/filter_stages.py (scale rule, fp16 pack, tile and bitmap layouts, keys, threshold rule,
error bounds, accumulation probes) against hand-built cases and exact rational arithmetic.  No GPU."""
import os
import sys
from fractions import Fraction

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import filter_stages as FS  # noqa: E402


def test_scale_rule_brings_the_largest_magnitude_into_2_14_2_15():
    rng = np.random.default_rng(0)
    bits = rng.integers(0, 0x7F800000, 20000, dtype=np.int64)
    bits = np.concatenate([bits, [0, 1, 0x007FFFFF, 0x06800000, 0x06FFFFFF, 0x07000000, 0x3F800000, 0x46800000,
                                  0x46FFFFFF, 0x47000000, 0x7F7FFFFF, 0x7F800000, 0x7FC00000]])
    e = FS.fp16_scale_exp(torch.from_numpy(bits)).numpy()
    for b, x in zip(bits, e):
        if (b >> 23) in (0, 255) or (b >> 23) < 14:
            assert x == 0, hex(b)                   # zero, subnormal, inf / NaN, or below 2^-113: scale 1
        else:
            m = Fraction(float(np.array([b], np.int64).astype(np.int32).view(np.float32)[0]))
            v = m * Fraction(2) ** int(x)
            assert Fraction(2 ** 14) <= v < Fraction(2 ** 15), hex(b)
    assert FS.fp16_scale_exp(torch.tensor([0x3F800000])).item() == 14          # 1.0 -> 2^14
    assert FS.fp16_scale_exp(torch.tensor([0x07000000])).item() == 127         # 2^-113 -> 2^14
    assert FS.fp16_scale_exp(torch.tensor([0x06FFFFFF])).item() == 0           # just below 2^-113: left as it is


def _fp16_rn(x: Fraction) -> Fraction:
    """Round to nearest even onto the fp16 grid (normal and subnormal; no overflow in these cases)."""
    if x == 0:
        return Fraction(0)
    s = -1 if x < 0 else 1
    a = abs(x)
    e = max(a.numerator.bit_length() - a.denominator.bit_length() - 1, -14)
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    while e > -14 and Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** (e - 10)
    n, r = divmod(a, q)
    if r * 2 > q or (r * 2 == q and n % 2 == 1):
        n += 1
    return s * n * q


def test_fp16_round_to_nearest_even_matches_exact_rounding():
    rng = np.random.default_rng(1)
    vals = list((rng.standard_normal(3000) * 2.0 ** rng.integers(-26, 15, 3000)).astype(np.float32))
    vals += [np.float32(1 + 2.0 ** -11), np.float32(1 + 3 * 2.0 ** -11), np.float32(2.0 ** -25), np.float32(3 * 2.0 ** -26),
             np.float32(2.0 ** -24 * 1.5), np.float32(-(2.0 ** 14) * (1 + 2.0 ** -11))]
    got = torch.tensor(np.array(vals, np.float32)).half().double().numpy()
    for v, g in zip(vals, got):
        assert Fraction(float(g)) == _fp16_rn(Fraction(float(v))), v


def test_pack_layout_places_each_element_by_hand():
    """[tile][k/8][16][8][8]: element (row, k) at tile row // 128, k block k // 8, core matrix (row % 128) // 8, row
    row % 8, position k % 8; rows beyond R and columns beyond d are zero; per-row scales."""
    R, d, KP, rows_pad = 130, 9, 32, 256
    x = torch.arange(1, R * d + 1, dtype=torch.float32).view(R, d)
    exps = torch.zeros(R, dtype=torch.int64)
    exps[129] = 3
    p = FS.pack_tiles(x, exps, KP, rows_pad).view(torch.float16)
    assert p.numel() == rows_pad * KP

    def at(row, k):
        return p[(((row // 128) * (KP // 8) + k // 8) * 16 + (row % 128) // 8) * 64 + (row % 8) * 8 + k % 8].item()
    assert at(0, 0) == 1 and at(1, 0) == 1 + d and at(0, 8) == 9
    assert at(129, 8) == (129 * d + 9) * 8
    assert at(127, 3) == float(torch.tensor(127 * d + 4.0).half())
    assert at(5, 9) == 0 and at(200, 0) == 0                          # K padding, padded rows
    back = FS.unpack_tiles(FS.pack_tiles(x, exps, KP, rows_pad), R, KP).float()
    want = torch.zeros(R, KP); want[:, :d] = (x * torch.ldexp(torch.ones(R), exps.float())[:, None]).half().float()
    assert torch.equal(back, want)


def test_bitmap_unpack_by_hand():
    w = np.zeros((1, 2, 4), np.uint32)
    w[0, 0, 0] = 1 << 31                        # column 0
    w[0, 0, 1] = 1                              # column 63
    w[0, 1, 3] = (1 << 31) | 1                  # columns 128 + 96, 128 + 127
    bits = FS.unpack_bitmap(torch.from_numpy(w.view(np.int32)), 2)
    assert torch.nonzero(bits[0]).flatten().tolist() == [0, 63, 224, 255]


def test_keys_and_threshold_rule():
    x = torch.tensor([-float("inf"), -2.0, -0.0, 0.0, 1e-45, 1.0, 3.0, float("inf")])
    k = FS.float_key(x)
    assert torch.all(k[1:] > k[:-1]) and int(k[0]) == 0x007FFFFF
    assert torch.equal(FS.key_float(k).view(torch.int32), x.view(torch.int32))
    g = torch.tensor([[5.0, 1.0, 3.0, -float("inf"), 2.0]])
    t, kth = FS.rule_threshold(g, torch.tensor([3]), 32)
    assert t.item() == 2.0 and kth.item() == 2.0
    g2 = torch.tensor([[1.0 + 2.0 ** -10, 1.0 + 2.0 ** -3, 7.0]])
    t16, kth = FS.rule_threshold(g2, torch.tensor([2]), 16)      # 16 key bits keep 7 significand bits
    assert kth.item() == 1.0 + 2.0 ** -3 and t16.item() == 1.0 + 2.0 ** -3
    t16, _ = FS.rule_threshold(g2, torch.tensor([3]), 16)
    assert t16.item() == 1.0                                    # lower edge of the bucket of 1 + 2^-10
    t24, _ = FS.rule_threshold(torch.tensor([[1.0 + 2.0 ** -20]]), torch.tensor([1]), 24)
    assert t24.item() == 1.0


def test_bound_constants_match_the_documented_values():
    assert abs(FS.knn_eps(4096) - 1.47e-3) < 5e-6                 # knn_cf.cu: "At F = 4096: eps = ... = 1.47e-3"
    assert FS.knn_steps(4100) == 260 and FS.knn_steps(200) == 16
    # K3: eps = 2^-10 (two roundings of 2^-11) + slack 2^-13 for the accumulation (S <= 8: 2^-17) and the fp32 chain
    assert FS.CF_EPS == 2.0 ** -10 + 2.0 ** -13
    assert FS.acc_bound(8, 1.0) + 128 * 2.0 ** -24 < FS.CF_EPS - 2.0 ** -10 - 2.0 ** -22


def _exp2(v: Fraction) -> int:
    """floor(log2 |v|), v != 0."""
    a = abs(v)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    while Fraction(2) ** e > a:
        e -= 1
    while Fraction(2) ** (e + 1) <= a:
        e += 1
    return e


def _trunc(v: Fraction, q: Fraction) -> Fraction:
    return (abs(v) // q) * q * (1 if v >= 0 else -1)


def _step_sum(c: Fraction, prods, guard: int, per_addend: bool) -> Fraction:
    """An adder model for one MMA step over the addends c, p_0 .. p_15: align to the largest one's exponent e and keep
    guard bits below its ulp 2^(e - 23).  per_addend: each addend is truncated to that grid, the sum is exact and is then
    truncated to 24 significant bits; otherwise only the exact sum is truncated, on the aligned grid."""
    addends = [c] + list(prods)
    if all(v == 0 for v in addends):
        return Fraction(0)
    q = Fraction(2) ** (max(_exp2(v) for v in addends if v != 0) - 23 - guard)
    if not per_addend:
        return _trunc(sum(addends, Fraction(0)), q)
    t = sum((_trunc(v, q) for v in addends), Fraction(0))
    return _trunc(t, Fraction(2) ** (_exp2(t) - 23)) if t != 0 else t


def _worst_ratio(a, b, guard, per_addend, one_step=False):
    """Worst error over the (row, item) pairs against the summed bound, or (one_step) against one step's."""
    K = a.shape[1]
    S = K // 16
    worst = 0.0
    for r in range(a.shape[0]):
        for g in range(b.shape[0]):
            p = [Fraction(float(a[r, k])) * Fraction(float(b[g, k])) for k in range(K)]
            c = Fraction(0)
            for s in range(S):
                c = _step_sum(c, p[16 * s:16 * s + 16], guard, per_addend)
            err = abs(c - sum(p, Fraction(0)))
            worst = max(worst, float(err / Fraction(FS.acc_bound(1 if one_step else S, float(sum(abs(v) for v in p))))))
    return worst


def _h100_step_ratio(n_small, g, carry):
    """One step of the measured adder (2 guard bits per addend, then a 24-bit truncation) on the worst-case operands of
    filter_stages.worst_rows: P = 2^28 and n_small products 2^(5 - g) (1 - 2^-11), in the same step or (carry) added to
    c = P in the next; returns the error / (2^-22 (|c| + sum |p|))."""
    P, small = Fraction(2 ** 28), Fraction(2) ** (5 - g) * (1 - Fraction(1, 2 ** 11))
    c, prods = (P, [small] * n_small) if carry else (Fraction(0), [P] + [small] * n_small)
    got = _step_sum(c, prods, guard=2, per_addend=True)
    total = c + sum(prods, Fraction(0))
    return float(abs(got - total) / (Fraction(2) ** -22 * total))


def test_measured_adder_model_reproduces_the_h100_and_stays_inside_the_step_bound():
    """tests/test_gpu_filter_stages.py's worst-case probes on an H100 SXM gave, per (label, g), the ratios below
    (err / 2^-22 (|c| + sum |p|)).  An adder that truncates each aligned addend 2 bits below the largest one's ulp and
    then the sum to 24 bits reproduces every one of them; its worst case, 16 addends just below the grid plus the final
    truncation, is < 5 x 2^-23 = 2.5 x 2^-22 -- inside the per-step term STEP_ERR = 2^-20 that knn_cf.cu now assumes.
    With one guard bit the same operands would reach 3.75 x 2^-22, with none 7.5: the probes tell them apart."""
    measured = {(3, 0, False): 0.499, (7, 0, False): 0.998, (15, 0, False): 1.996, (15, 0, True): 1.996,
                (3, 1, False): 0.750, (7, 1, False): 1.249, (15, 1, False): 2.248, (15, 1, True): 2.248,
                (3, 2, False): 0.375, (7, 2, False): 0.875, (15, 2, False): 1.874, (15, 2, True): 1.874,
                (3, 3, False): 0.187, (7, 3, False): 0.437, (15, 3, False): 0.937, (15, 3, True): 0.937}
    for (n, g, carry), want in measured.items():
        assert abs(_h100_step_ratio(n, g, carry) - want) < 1.5e-3, (n, g, carry)
    # the model's worst case over the grid: 16 addends a hair below 2^(e - 25) multiples, next to a top of 2^e
    eps = Fraction(1, 2 ** 11)
    top = Fraction(2 ** 28)
    for k in (1, 2, 3):
        small = Fraction(2) ** (5 - 2) * (k - eps)
        worst = _step_sum(top, [small] * 16, guard=2, per_addend=True)
        total = top + 16 * small
        assert abs(worst - total) < 5 * Fraction(2) ** -23 * total
    assert 2.5 * 2.0 ** -22 < FS.STEP_ERR
    one_guard = _step_sum(Fraction(0), [top] + [Fraction(2) ** 4 * (1 - eps)] * 15, guard=1, per_addend=True)
    assert abs(one_guard - top - 15 * Fraction(2) ** 4 * (1 - eps)) / (Fraction(2) ** -22 * top) > 3.7


def test_accumulation_bound_holds_for_the_assumed_adder_and_the_probes_catch_a_weaker_one():
    """Exact rationals: the measured adder (2 guard bits per addend) stays within the summed bound on every random probe
    family; one that truncates each aligned addend with no guard bit exceeds one step's bound on the worst-case operands
    -- so the GPU probes can tell the two apart."""
    K = 32
    b = FS.probe_items(4, K, seed=2)
    for fam in range(4):
        a = FS.probe_rows(4, K, seed=fam, family=fam)
        assert torch.equal(a.half().float(), a) and torch.equal(b.half().float(), b)          # fp16-exact operands
        m = FS.absmax_bits(a)
        assert torch.all(FS.fp16_scale_exp(m) == 0) and torch.all(FS.fp16_scale_exp(FS.absmax_bits(b).max()[None]) == 0)
        assert _worst_ratio(a, b, guard=2, per_addend=True) <= 1.0
        if fam == 1:
            assert _worst_ratio(a, b, guard=2, per_addend=True, one_step=True) <= 1.0
    aw, _, _ = FS.worst_rows(64, K)
    bw = FS.worst_items(4, K)
    assert torch.equal(aw.half().float(), aw) and torch.equal(bw.half().float(), bw)
    assert _worst_ratio(aw[2:32:4], bw, guard=2, per_addend=True, one_step=True) <= 1.0
    assert _worst_ratio(aw[2:32:4], bw, guard=0, per_addend=True, one_step=True) > 1.0
