"""Host restatements of the certified filters' intermediate stages (K3 csrc/score_cf.cu, K7 csrc/knn_cf.cu), for
tests/test_gpu_filter_stages.py: the power-of-two scale rule and fp16 pack of the operands, the tile layout, the bitmap
layout, the order-preserving keys, the threshold rule and the error bounds.  Everything here is torch (device or CPU)
and is checked on the CPU against hand-built cases and exact rational arithmetic in tests/test_filter_stages_host.py."""
import math

import torch

TILE = 128                      # rows of an operand tile, both filters
CF_EPS = 1.125 / 1024           # K3: |s~ - s| <= CF_EPS |u| max|i| + subnormal term (score_cf.cu)
CF_EPS_SUB = 2.0 ** -24
CF_THR_BITS = 16                # K3: threshold search on the top 16 key bits while G <= 1024
KN_KC = 64                      # K7: K padded to a multiple of 64
KN_GROUP = 16
KN_THR_BITS = 24                # K7: radix select over the top 24 key bits


# ---------------------------------------------------------------------------------------------- scale rule and pack
def fp16_scale_exp(m_bits):
    """fp16_scale_for (tc_common.cuh): the exponent e of the power of two that brings a largest magnitude (its fp32 bit
    pattern, int tensor) into [2^14, 2^15); 0 for a zero, inf / NaN, or a magnitude below 2^-113."""
    e = (torch.as_tensor(m_bits).to(torch.int64) >> 23) & 0xFF
    ok = (e != 0) & (e != 255) & (e >= 14)
    return torch.where(ok, 141 - e, torch.zeros_like(e))


def absmax_bits(x):
    """Largest |element| of each row of fp32 x [R, d] as a bit pattern (NaN above inf above every finite value)."""
    return (x.contiguous().view(torch.int32).to(torch.int64) & 0x7FFFFFFF).amax(dim=1)


def pack_tiles(x, exps, KP, rows_pad):
    """fp16(RN) of x [R, d] (fp32) times 2^exps (per row [R], or one value), zero-padded to [rows_pad, KP], in the
    canonical K-major no-swizzle wgmma layout [tile][KP/8][16][8][8] (store_fp16x8).  Returns int16 [rows_pad * KP]."""
    R, d = x.shape
    exps = torch.as_tensor(exps, device=x.device).to(torch.int64).expand(R)
    sc = torch.ldexp(torch.ones(R, dtype=torch.float32, device=x.device), exps.to(torch.float32))
    full = torch.zeros(rows_pad, KP, dtype=torch.float32, device=x.device)
    full[:R, :d] = x * sc[:, None]                         # a power of two: exact in fp32 barring under / overflow
    h = full.half().view(torch.int16)
    h = h.view(rows_pad // TILE, 16, 8, KP // 8, 8).permute(0, 3, 1, 2, 4)
    return h.contiguous().view(-1)


def unpack_tiles(packed, rows, KP):
    """Inverse of pack_tiles: int16 [tiles * 128 * KP] -> fp16 [tiles * 128, KP], rows in order; first `rows` rows."""
    t = packed.view(-1, KP // 8, 16, 8, 8).permute(0, 2, 3, 1, 4).contiguous()
    return t.view(-1, KP)[:rows].view(torch.float16)


def unpack_bitmap(words, n_it):
    """The pass-2 bitmap [R, n_it] x uint4 (int32 [R, n_it, 4]) -> bool [R, n_it * 128]: bit (31 - c) of word b is
    column 32 b + c of the item tile."""
    w = words.view(-1, n_it, 4, 1).to(torch.int64) & 0xFFFFFFFF
    sh = torch.arange(31, -1, -1, device=words.device, dtype=torch.int64)
    return ((w >> sh) & 1).bool().view(-1, n_it * TILE)


# ---------------------------------------------------------------------------------------------- keys and threshold rule
def float_key(x):
    """common.cuh float_key of fp32 x as int64 in [0, 2^32): ascending key = ascending value."""
    b = x.contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    return torch.where(b >= 0x80000000, 0xFFFFFFFF - b, b | 0x80000000)


def key_float(k):
    k = torch.as_tensor(k).to(torch.int64)
    b = torch.where(k >= 0x80000000, k & 0x7FFFFFFF, 0xFFFFFFFF - k)
    return torch.where(b >= 0x80000000, b - (1 << 32), b).to(torch.int32).view(torch.float32)


def rule_threshold(g, need, bits):
    """The threshold the filters take for each row of group maxima g [R, G] (fp32) and rank need [R] (1 <= need <= G):
    the need-th largest key with its low 32 - bits bits cleared (the lower edge of its bucket; bits = 32: the value).
    Returns (t fp32 [R], the need-th largest maximum fp32 [R])."""
    keys = float_key(g)
    kth = keys.sort(dim=1, descending=True).values.gather(1, (need.to(torch.int64) - 1)[:, None])[:, 0]
    mask = ((1 << 32) - 1) ^ ((1 << (32 - bits)) - 1)
    return key_float(kth & mask), key_float(kth)


# ---------------------------------------------------------------------------------------------- bounds
STEP_ERR = 2.0 ** -20            # one m64n128k16 step: error <= STEP_ERR (|c| + sum |p|) (knn_cf.cu, ERROR BOUND (2))


def acc_bound(S, abs_sum):
    """The accumulation term of both files: S m64n128k16 steps, each adding its exact products with error at most
    STEP_ERR (|c| + sum |p|), summed: S STEP_ERR (1 + 2^-9) sum_k |a^_k b^_k|."""
    return S * STEP_ERR * (1 + 2.0 ** -9) * abs_sum


def cf_eps_prime(un, mn, d):
    """K3 (cf_thr_kernel), per row: |s~ - s| <= eps' = CF_EPS un mn + 2^-24 sqrt(d) (un + mn + 1), scaled domain;
    thr = t - 2 eps'.  un, mn: the kernel's (rounded-up) row norm and largest item norm."""
    return CF_EPS * un * mn + CF_EPS_SUB * math.sqrt(d) * (un + mn + 1.0)


def knn_steps(F):
    return -(-F // KN_KC) * (KN_KC // 16)


def knn_eps(F):
    """K7 eps(F) = 2^-10 + 2^-22 + (S STEP_ERR + F 2^-24)(1 + 2^-9), S = F_pad / 16 (knn_cf.cu, ERROR BOUND)."""
    return 2.0 ** -10 + 2.0 ** -22 + (knn_steps(F) * STEP_ERR + F * 2.0 ** -24) * (1 + 2.0 ** -9)


def knn_eps_prime(un, mn, F, sc):
    """K7 cosine route, per query row: eps' = eps(F) un mn + sub(F) in the scaled domain (un, mn scaled norms);
    thr = t - 2 eps' (1 + 2^-8)."""
    return knn_eps(F) * un * mn + 2.0 ** -25 * math.sqrt(F) * (un + mn) + F * 2.0 ** -50 + F * 2.0 ** -149 * sc * sc


def knn_shrink_e(A, nq, Bm, Rmax, nmin, nmax, shrink, F, sc):
    """K7 shrink route (knn_thr_kernel<true>), per query row, in exact arithmetic: the bound e on |v~ - v|, v = s / D;
    thr = t - 2 e (1 + 2^-8).  A = rnorm[q], nq = norms[q], Bm = the largest rnorm, Rmax = max rnorm[i] / norms[i],
    nmin / nmax = the smallest / largest norms[i], all unscaled."""
    eps = knn_eps(F)
    fac = nq * nmax / (nq * nmax + shrink)
    RR = (0.0 if A == 0 else A / nq) * Rmax * fac
    Dmin = nq * nmin + shrink
    isc = 1.0 / sc
    sub = (2.0 ** -25 * math.sqrt(F) * (A + Bm) * isc + F * 2.0 ** -50 * isc * isc + 2.0 ** -120) / Dmin
    vmax = RR * (1 + 2 * eps) + sub
    return eps * RR + sub + 2.0 ** -23 * vmax


# ---------------------------------------------------------------------------------------------- adversarial probes
def probe_rows(R, K, seed, family):
    """Operands for the accumulation probe: rows [R, K] of fp16-exact fp32 values whose largest element lies in
    [2^14, 2^15) (the scale rule leaves them as they are) and whose products with probe_items stress an adder that
    aligns to the largest exponent and truncates.  Per K step of 16 (slot 0 of the step = the big element):
      0  every step: one big product plus 15 products just below the fp32 ulp of the big one;
      1  the same in one step only (r mod S); every other step is zero: the error of a single step;
      2  big products of alternating sign (+P, -P, ...: exact cancellation across steps) plus the small ones;
      3  exponents spread over the whole scaled fp16 range, one big element in step 0."""
    g = torch.Generator().manual_seed(seed)
    S = K // 16
    a = torch.zeros(R, S, 16, dtype=torch.float64)
    mant = 1 + torch.randint(0, 1024, (R, S, 16), generator=g).double() / 1024
    big = 2.0 ** 14 * (1 + torch.randint(0, 1024, (R, 1), generator=g).double() / 1024)
    if family in (0, 2):
        a[:, :, 0] = big
        a[:, :, 1:] = 4 * mant[:, :, 1:]
        if family == 2:
            a[:, 1::2, 0] *= -1
    elif family == 1:
        s = torch.arange(R) % S
        a[torch.arange(R), s, 0] = big[:, 0]
        a[torch.arange(R), s, 1:] = 4 * mant[torch.arange(R), s, 1:]
    else:
        e = torch.randint(-12, 13, (R, S, 16), generator=g).double()
        a[:] = torch.ldexp(mant, e.to(torch.int64))
        a[:, 0, 0] = big[:, 0]
        a[:, 1:, 0] = 0
    return a.view(R, K).float()


def probe_items(G, K, seed):
    """The probe items [G, K]: slot 0 of every step 2^14 (1 + m / 1024), the other slots powers of two 2^-1 .. 2^2, so
    that against probe_rows the small products land 1 .. 4 binades below the fp32 ulp of the big one."""
    g = torch.Generator().manual_seed(seed)
    S = K // 16
    b = torch.ldexp(torch.ones(G, S, 16, dtype=torch.float64), torch.randint(-1, 3, (G, S, 16), generator=g))
    b[:, :, 0] = 2.0 ** 14 * (1 + torch.randint(0, 1024, (G, 1), generator=g).double() / 1024)
    return b.view(G, K).float()


WORST = ("3 below-granularity products", "7 below-granularity products", "15 below-granularity products",
         "15 below the accumulator's ulp")


def worst_rows(R, K):
    """Operands for the worst case of an adder that truncates at several points (per product or per partial sum): one
    large product P = 2^14 * 2^14 = 2^28, at the bottom of its binade (fp32 ulp 2^5), and small products each just below
    a power of two, 2^e (1 - 2^-11), so that with g guard bits every one of them falls just short of the truncation
    granularity 2^(5 - g) when e = 5 - g.  Against worst_items (slot 0 of a step 2^14, the other slots 2^y, y = item mod 4)
    row r carries 2^x (2 - 2^-10), x = -3 + (r / 4) mod 8, so e = x + y + 1 sweeps -2 .. 8 (g = 7 .. -3) over the items.
    Label r mod 4: 0 / 1 / 2 = P and 3 / 7 / 15 small products in the same step (one partial group of 4 or 8, or the
    whole step), every other step zero; 3 = P alone in one step and 15 small products in the next (c = P when they are
    added).  The step is (r / 32) mod S.  Returns (rows [R, K] fp32, label [R], x [R])."""
    S = K // 16
    a = torch.zeros(R, S, 16, dtype=torch.float64)
    r = torch.arange(R)
    lab, x, s = r % 4, -3 + (r // 4) % 8, (r // 32) % S
    small = torch.ldexp(torch.full((R,), 2 - 2.0 ** -10, dtype=torch.float64), x)
    for i in range(R):
        n = (3, 7, 15, 15)[lab[i]]
        s0 = int(s[i]) if lab[i] < 3 else int(s[i]) % (S - 1)
        a[i, s0, 0] = 2.0 ** 14
        a[i, s0 + (lab[i] == 3), 1:n + 1] = small[i]
    return a.view(R, K).float(), lab, x


def worst_items(G, K):
    S = K // 16
    b = torch.ldexp(torch.ones(G, S, 16, dtype=torch.float64), (torch.arange(G) % 4)[:, None, None].expand(G, S, 16))
    b[:, :, 0] = 2.0 ** 14
    return b.view(G, K).float()
