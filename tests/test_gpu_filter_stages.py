"""The certified filters' intermediate stages against float64, stage by stage: the fused scoring (K3, csrc/score_cf.cu)
and the kNN build (K7, csrc/knn_cf.cu).  The end-to-end tests (test_gpu_score_exact.py, test_gpu_knn.py) cannot see a pass
that overestimates (more candidates, same result), a small underestimate outside the top-k, or disagreement between K3's
two passes; these tests read the scratch back after a call and check each stage on its own:

  packs     fp16_RN(2^e x) bit for bit in the wgmma tile layout, e per user row / one for the catalogue or table; norms
            and headers are upper bounds, tight to their documented rounding;
  pass 1    every group maximum within the accumulation term of max(a^ . b^) over the group's real items (float64 of the
            fp16 operands the tensor cores were given), and within the documented eps' of the exact score; groups past
            the last item exactly -inf;
  threshold thr <= t - 2 eps' and not vacuous (>= t - 3 eps'), t the documented rule on the kernel's maxima; and the
            threshold the kernel implies, thr + 2 eps', has need maxima at or above it (t itself is never stored, so
            the rule's own properties, >= need maxima >= t and t <= the need-th largest, only restate the rule);
  pass 2    (K3) tolerance-free against pass 1: a bit set in a group <=> the group's maximum >= thr; no bit past the last
            item; items clear of thr by more than the accumulation term set / unset accordingly; every member of the exact
            top-k set;
  flags     (K3) each row's reason equals the one derived from the stages above.
A last part measures the accumulation assumption both bounds rest on, on adversarial operands: random families
(filter_stages.probe_rows) and the worst case of a truncating adder (filter_stages.worst_rows).

The scratch offsets come from mmrec_debug_cf_scratch / mmrec_debug_knn_scratch, not from a restated layout.  Only the last
row block's scratch survives a call, and nothing after the stages read here rewrites them: K3's cf_final_kernel reads the
bitmap and writes only flags (its reasons 4 / 8, into rows pass 1 left at 0), the counter and row_of_slot; cf_exact_kernel
writes its own key buffer and the output.  K7's knn_final_kernel reads gmax / thr / flags and writes the counter, the
fallback lists and the output; the exact route uses its own region.  K7 is called through the C ABI with a workspace of
the test's own, because ops.knn_topk drops its scratch.  The workspace is filled with 0xFF first, so that bytes no stage
may write (padded user rows, the slack behind each region) can be checked untouched."""
import os
import sys

import pytest
import torch

from oracle import mmrec_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import filter_stages as FS  # noqa: E402

pytestmark = pytest.mark.gpu
SENT = 0xFF


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def _layout(fn, *args, n):
    import ctypes
    out = (ctypes.c_int64 * n)()
    assert fn(*args, ctypes.addressof(out), n) == n
    return list(out)


def _region(ws, o0, off, nbytes, dtype):
    return ws[o0 + off:o0 + off + nbytes].view(dtype)


def _chunks(rows, cols, budget=1 << 25):
    step = max(1, budget // max(cols, 1))
    return [(r, min(rows, r + step)) for r in range(0, rows, step)]


# ================================================================================================ K3
class CfRun:
    pass


def cf_run(ue, ie, users, mask, k, in_call):
    """One fused call on a 0xFF-filled workspace of the test's own; returns the scratch views of the last row block."""
    from mmrec_b200 import _lib, ops
    lib = _lib.load()
    dev = ue.device
    B = ue.shape[0] if users is None else users.numel()
    I, d = ie.shape
    nnz = 0 if mask is None else mask.shape[1]
    L = _layout(lib.mmrec_debug_cf_scratch, B, I, d, k, nnz, int(in_call), n=16)
    r = CfRun()
    (r.rows_blk, r.rows_pad, r.KP, r.gw, r.n_it, r.G, r.G_valid, off_cat, r.hdr_bytes, off_upk, off_unorm, off_gmax,
     off_thr, off_bitmap, off_flags, total) = L
    ws = torch.full((max(lib.mmrec_score_topk_workspace_bytes(B, I, d, k) + 4 * nnz + 4096, total + 1024),), SENT,
                    dtype=torch.uint8, device=dev)
    o0 = (-ws.data_ptr()) % 1024
    cat, cat_ptr = None, None
    cat_bytes = lib.mmrec_catalog_bytes(I, d)
    if not in_call:
        cat = torch.full((cat_bytes + 1024,), SENT, dtype=torch.uint8, device=dev)
        c0 = (-cat.data_ptr()) % 1024
        cat_ptr = cat.data_ptr() + c0
        ops.check(lib.mmrec_catalog_pack_f32(I, ie.data_ptr(), d, d, cat_ptr, cat_bytes, ops._stream()), "catalog_pack")
        r.cat = cat[c0:c0 + cat_bytes]
    idx = torch.empty(B, k, dtype=torch.int64, device=dev)
    val = torch.empty(B, k, device=dev)
    mr = mask[0].contiguous() if nnz else None
    mc = mask[1].contiguous() if nnz else None
    ops.set_score_path("fused")
    try:
        ops.check(lib.mmrec_score_topk_cat_f32(B, users.data_ptr() if users is not None else None, ue.data_ptr(), d, I,
                                               ie.data_ptr(), d, d, cat_ptr, nnz, mr.data_ptr() if nnz else None,
                                               mc.data_ptr() if nnz else None, k, 0, idx.data_ptr(), val.data_ptr(),
                                               ws.data_ptr(), ws.numel(), ops._stream()), "score_topk_cat")
    finally:
        ops.set_score_path("auto")
    torch.cuda.synchronize()
    if in_call:
        r.cat = _region(ws, o0, off_cat, cat_bytes, torch.uint8)
    r.hdr = r.cat[:r.hdr_bytes].view(torch.int32)
    r.ipk = r.cat[r.hdr_bytes:].view(torch.int16)
    r.r0 = (B - 1) // r.rows_blk * r.rows_blk
    r.nb = B - r.r0
    r.upk = _region(ws, o0, off_upk, r.rows_pad * r.KP * 2, torch.int16)
    r.unorm_all = _region(ws, o0, off_unorm, r.rows_pad * 4, torch.float32)
    r.gmax = _region(ws, o0, off_gmax, r.rows_blk * r.G * 4, torch.float32).view(r.rows_blk, r.G)
    r.gmax_slack = ws[o0 + off_gmax + r.rows_blk * r.G * 4:o0 + off_thr]
    r.thr_all = _region(ws, o0, off_thr, r.rows_pad * 4, torch.float32)
    r.bitmap = _region(ws, o0, off_bitmap, r.rows_blk * r.n_it * 16, torch.int32).view(r.rows_blk, r.n_it, 4)
    r.bitmap_slack = ws[o0 + off_bitmap + r.rows_blk * r.n_it * 16:o0 + off_flags]
    r.flags = _region(ws, o0, off_flags, (r.rows_blk + 1) * 4, torch.int32)
    r.idx, r.val = idx, val
    return r


def cf_same_scratch(a, b):
    """Catalog and in-call packing leave the same bits in every stage."""
    assert torch.equal(a.cat, b.cat), "catalogue bytes differ between Catalog and in-call packing"
    for name in ("upk", "unorm_all", "thr_all", "flags"):
        assert torch.equal(getattr(a, name).view(torch.uint8), getattr(b, name).view(torch.uint8)), name
    assert torch.equal(a.idx, b.idx), "indices"
    nb = a.nb
    assert torch.equal(a.gmax[:nb].view(torch.int32), b.gmax[:nb].view(torch.int32)), "gmax"
    assert torch.equal(a.bitmap[:nb], b.bitmap[:nb]), "bitmap"
    assert torch.equal(a.val.view(torch.int32), b.val.view(torch.int32)), "values"


def cf_check_stages(r, ue, ie, users, mask, k):
    dev = ue.device
    U_all = ue if users is None else ue[users]
    U = U_all[r.r0:]
    nb, KP, G, Gv, n_it = r.nb, r.KP, r.G, r.G_valid, r.n_it
    I, d = ie.shape
    S = KP // 16
    w = 16 * r.gw
    fin = torch.isfinite(U).all(dim=1)
    # ---- packs, norms, header
    eu = FS.fp16_scale_exp(FS.absmax_bits(U))
    nb_pad = -(-nb // 256) * 256                           # the block's tile pairs (rows beyond: an earlier block's)
    assert torch.equal(r.upk[:nb_pad * KP], FS.pack_tiles(U, eu, KP, nb_pad)), "user pack"
    hdr = r.hdr.cpu().to(torch.int64)
    assert hdr[4].item() == FS.absmax_bits(ie).max().item(), "catalogue largest |element|"
    assert hdr[1:4].tolist() == [I, d, KP] and not hdr[5:].any(), "catalogue header"
    ei = FS.fp16_scale_exp(hdr[4:5]).item()
    assert torch.equal(r.ipk, FS.pack_tiles(ie, torch.tensor([ei]), KP, n_it * FS.TILE)), "catalogue pack"
    su = torch.ldexp(torch.ones(nb, dtype=torch.float64, device=dev), eu.double())
    un_true = (U.double() * su[:, None]).norm(dim=1)
    unorm = r.unorm_all[:nb].double()
    ok = fin & (un_true > 0)
    assert torch.all(unorm[ok] >= un_true[ok]) and torch.all(unorm[ok] <= un_true[ok] * (1 + 2e-6)), "user row norms"
    assert torch.all(unorm[fin & (un_true == 0)] == 0)
    first = r.rows_blk if r.r0 else nb                     # rows an earlier block wrote
    assert torch.all(r.unorm_all[first:].view(torch.uint8) == SENT) and \
        torch.all(r.thr_all[first:].view(torch.uint8) == SENT), "padded user rows were written"
    assert torch.all(r.gmax_slack == SENT) and torch.all(r.bitmap_slack == SENT), "writes past the last row"
    mn = torch.tensor(hdr[0].item(), dtype=torch.int32).view(torch.float32).item()
    mn_true = (ie.double() * 2.0 ** ei).norm(dim=1).max().item()
    assert mn_true <= mn <= mn_true * (1 + 2e-6), "largest item norm"
    # ---- need, flags 1 / 2, threshold rule
    need = torch.full((nb,), k, dtype=torch.int64, device=dev)
    if mask is not None:
        mr = mask[0] - r.r0
        need += torch.bincount(mr[(mr >= 0) & (mr < nb)], minlength=nb)
    gmax = r.gmax[:nb]
    flag1 = need > Gv
    bits_rule = 16 if G <= 1024 else 32
    t, kth = FS.rule_threshold(gmax, need.clamp(max=G), bits_rule)
    flag2 = ~flag1 & ~(torch.isfinite(t) & torch.isfinite(r.unorm_all[:nb]))
    served = ~flag1 & ~flag2
    thr = r.thr_all[:nb].double()
    assert torch.all(torch.isinf(thr[~served])), "flagged rows keep thr = +inf"
    t64 = t.double()
    epsp = FS.cf_eps_prime(unorm, mn, d)
    # (the two rule asserts restate the documented rule on the kernel's own maxima; the kernel never stores t)
    cnt_ge = (gmax[:, :Gv] >= t[:, None]).sum(1)
    assert torch.all(cnt_ge[served] >= need[served]), "fewer than need maxima >= t"
    assert torch.all(t[served] <= kth[served]), "t above the need-th largest maximum"
    # the kernel's thr: within [t - 3 eps', t - 2 eps' + the rounding of its fp32 margin and subtraction], and the t it
    # implies, thr + 2 eps' less that rounding, still has need maxima at or above it (the certificate itself)
    slack = 2.0 ** -21 * epsp + 2.0 ** -23 * t64.abs()
    assert torch.all((thr <= t64 - 2 * epsp + slack)[served]), "thr above t - 2 eps'"
    assert torch.all((thr >= t64 - 3 * epsp)[served]), "thr below t - 3 eps': the margin is vacuous"
    implied = ((gmax[:, :Gv].double() >= (thr + 2 * epsp - slack)[:, None]).sum(1))
    assert torch.all(implied[served] >= need[served]), "fewer than need maxima at or above thr + 2 eps'"
    # ---- pass 1 and pass 2 against float64, in row chunks
    A = FS.unpack_tiles(r.upk, nb, KP).double()
    Bi = FS.unpack_tiles(r.ipk, I, KP).double()
    bits = FS.unpack_bitmap(r.bitmap[:nb], n_it)
    assert not bits[:, I:].any(), "bit set past the last item"
    gb = bits.view(nb, G, w).any(-1)
    ge = gmax >= r.thr_all[:nb, None]
    assert torch.equal(gb[served], ge[served]), "pass 2 bits disagree with pass 1 maxima against thr"
    assert not bits[flag1].any()
    npad = n_it * FS.TILE - I
    for c0, c1 in _chunks(nb, n_it * FS.TILE):
        f = served[c0:c1]
        dot = A[c0:c1] @ Bi.T
        absd = A[c0:c1].abs() @ Bi.abs().T
        tol = FS.acc_bound(S, absd)
        gm = torch.nn.functional.pad(dot, (0, npad), value=-float("inf")).view(c1 - c0, G, w).amax(-1)
        ga = torch.nn.functional.pad(absd, (0, npad)).view(c1 - c0, G, w).amax(-1)
        gk = gmax[c0:c1].double()
        assert torch.all(gk[:, Gv:] == -float("inf")), "groups past the last item must be -inf"
        err = (gk[:, :Gv] - gm[:, :Gv]).abs()
        bad = (err > FS.acc_bound(S, ga[:, :Gv])) & fin[c0:c1, None]
        assert not bad.any(), f"pass 1: {int(bad.sum())} group maxima outside the accumulation term of float64, worst " \
                              f"{float((err / FS.acc_bound(S, ga[:, :Gv]))[fin[c0:c1]].max()):.3g}"
        # the documented bound against the exact score (fp32 chain: within 16 2^-24 |u| max|i| of the real product)
        sc = su[c0:c1, None] * 2.0 ** ei
        s = (U[c0:c1].double() @ ie.double().T) * sc
        gs = torch.nn.functional.pad(s, (0, npad), value=-float("inf")).view(c1 - c0, G, w).amax(-1)[:, :Gv]
        gamma = 16 * 2.0 ** -24 * unorm[c0:c1, None] * mn + 192 * 2.0 ** -149 * sc
        bad = ((gk[:, :Gv] - gs).abs() + gamma > epsp[c0:c1, None]) & fin[c0:c1, None]
        assert not bad.any(), "pass 1 outside eps' of the exact score"
        th = thr[c0:c1, None]
        b = bits[c0:c1, :I]
        assert not (f[:, None] & (dot - tol >= th) & ~b).any(), "an item clear above thr has no bit"
        assert not (f[:, None] & (dot + tol < th) & b).any(), "an item clear below thr has a bit"
    # ---- every member of the exact top-k has its bit
    ub = (users if users is not None else torch.arange(ue.shape[0], device=dev))[r.r0:]
    ms = None
    if mask is not None:
        keep = (mask[0] >= r.r0)
        ms = torch.stack([mask[0][keep] - r.r0, mask[1][keep]])
    rv, ri = O.cf_exact_topk(ue, ie, ub, ms, k, device=dev)
    ri, rv = ri.to(dev), rv.to(dev)
    real = (rv != O.MASKED_SCORE) & served[:, None]
    hit = bits.gather(1, ri.clamp(max=I - 1))
    assert torch.all(hit[real]), "a member of the exact top-k has no bit"
    # ---- flags: the reason of each row
    pc = bits.sum(1)
    masked_in = torch.zeros(nb, dtype=torch.int64, device=dev)
    if ms is not None:
        okm = (ms[0] < nb) & (ms[1] >= 0) & (ms[1] < I)
        key = torch.unique(ms[0][okm] * I + ms[1][okm])
        rr, cc = key // I, key % I
        masked_in.index_add_(0, rr, bits[rr, cc].to(torch.int64))
    want = torch.where(flag1, 1, torch.where(flag2, 2, torch.where(pc > 512, 4, torch.where(pc - masked_in < k, 8, 0))))
    got = r.flags[:nb].to(torch.int64)
    assert torch.equal(got, want), f"flags differ in {int((got != want).sum())} rows"
    assert int(r.flags[r.rows_blk]) == int((want != 0).sum()), "counter"
    return want


def _mask(dev, B, I, kind, g, U=None, ie=None, k=0, Gv=0):
    if kind is None:
        return None
    r = torch.randint(0, B, (B * 4,), generator=g)
    c = torch.randint(0, I, (B * 4,), generator=g)
    rows, cols = [r, torch.tensor([-1, B])], [c, torch.tensor([1, 2])]
    if kind == "heavy":
        for row, n in [(0, Gv - k + 1), (min(1, B - 1), Gv - k)]:
            rows.append(torch.full((n,), row)); cols.append(torch.randperm(I, generator=g)[:n])
        top = (U[2 % B:2 % B + 1].double() @ ie.double().T).topk(min(100, I)).indices.cpu()[0]
        rows.append(torch.full((top.numel(),), 2 % B)); cols.append(top)
    m = torch.stack([torch.cat(rows), torch.cat(cols)])
    if kind == "sorted":
        m = m[:, torch.argsort(m[0], stable=True)]
    else:
        m = m[:, torch.randperm(m.shape[1], generator=g)]
    return m.to(dev)


def _tables(dev, B, I, d, mags, g):
    ue = torch.randn(B, d, generator=g) * 0.1
    ie = torch.randn(I, d, generator=g) * 0.1
    if mags == "mixed":
        ue *= torch.pow(10.0, torch.empty(B, 1).uniform_(-20, 20, generator=g))
    if mags == "special":
        ue[3] *= 1e-24                   # 1e-25-scale rows
        ue[4] *= 1e-24
        ue[5] = 0.0                      # zero row: every item ties at 0
        ue[6, 0] = float("inf")          # non-finite row
    return ue.to(dev), ie.to(dev)


CF_CASES = [
    # id, B, I, d, k, mask, magnitudes, users
    ("I7000-d64-B257", 257, 7000, 64, 50, "sorted", "plain", True),
    ("I16384-d32-B255", 255, 16384, 32, 50, "unsorted", "plain", False),
    ("I16385-d33-B256", 256, 16385, 33, 50, None, "mixed", False),
    ("I32769-d65-B1", 1, 32769, 65, 1, "sorted", "plain", False),
    ("I65537-d128-B257-heavy", 257, 65537, 128, 50, "heavy", "plain", True),
    ("I131073-d64-radix", 255, 131073, 64, 50, "unsorted", "mixed", False),
    ("I20001-d1", 257, 20001, 1, 20, "sorted", "plain", False),
    ("I7001-d128-B4097-special", 4097, 7001, 128, 50, "sorted", "special", False),
    ("k1-G2k-I129", 64, 129, 32, 1, "sorted", "plain", False),
    ("k50-G2k-I1537", 300, 1537, 64, 50, "heavy", "plain", False),
    ("k256-G2k-I8065", 256, 8065, 64, 256, "unsorted", "plain", False),
]


@pytest.mark.parametrize("case", CF_CASES, ids=[c[0] for c in CF_CASES])
def test_cf_stages(dev, case):
    _, B, I, d, k, mk, mags, with_users = case
    g = torch.Generator().manual_seed(B * 7 + I + d)
    ue, ie = _tables(dev, B + (50 if with_users else 0), I, d, mags, g)
    users = torch.randperm(ue.shape[0], generator=g)[:B].to(dev) if with_users else None
    from mmrec_b200 import _lib
    Gv = _layout(_lib.load().mmrec_debug_cf_scratch, B, I, d, k, 0, 1, n=16)[6]
    U = ue if users is None else ue[users]
    mask = _mask(dev, B, I, mk, g, U, ie, k, Gv)
    a = cf_run(ue, ie, users, mask, k, in_call=True)
    b = cf_run(ue, ie, users, mask, k, in_call=False)
    cf_same_scratch(a, b)
    flags = cf_check_stages(a, ue, ie, users, mask, k)
    if mags == "special":
        assert flags[6] == 2 and flags[5] == 4          # the non-finite row; the zero row (all items tie)


def test_cf_stages_two_row_blocks(dev):
    """1 000 003 items: the group maxima + bitmap exceed 512 MB, the batch runs as two row blocks; the second (257 rows,
    an odd user-tile pair) is the one left in the scratch."""
    from mmrec_b200 import _lib
    I, d, k = 1_000_003, 32, 50
    L = _layout(_lib.load().mmrec_debug_cf_scratch, 4096, I, d, k, 0, 1, n=16)
    B = L[0] + 257
    g = torch.Generator().manual_seed(99)
    ue, ie = _tables(dev, B, I, d, "plain", g)
    mask = _mask(dev, B, I, "sorted", g)
    a = cf_run(ue, ie, None, mask, k, in_call=True)
    assert a.r0 == L[0] and a.nb == 257
    cf_check_stages(a, ue, ie, None, mask, k)


# ================================================================================================ K7
class KnnRun:
    pass


def knn_run(X, rows, k, norms=None, shrink=0.0):
    from mmrec_b200 import _lib, ops
    lib = _lib.load()
    n, F = X.shape
    m = n if rows is None else rows.numel()
    L = _layout(lib.mmrec_debug_knn_scratch, n, F, m, k, n=15)
    r = KnnRun()
    (r.rows_blk, r.rows_pad, r.KP, grp, r.n_it, r.G, r.G_valid, off_hdr, off_xpk, off_rnorm, off_qpk, off_gmax, off_thr,
     off_flags, total) = L
    assert grp == FS.KN_GROUP
    ws = torch.full((lib.mmrec_knn_topk_workspace_bytes(n, F, m, k) + 1024,), SENT, dtype=torch.uint8, device=X.device)
    o0 = (-ws.data_ptr()) % 1024
    assert o0 + total - 1024 <= ws.numel()
    idx = torch.empty(m, k, dtype=torch.int64, device=X.device)
    val = torch.empty(m, k, device=X.device)
    rp = rows.data_ptr() if rows is not None else None
    if norms is None:
        rc = lib.mmrec_knn_topk_f32(n, X.data_ptr(), F, F, m, rp, k, idx.data_ptr(), val.data_ptr(), ws.data_ptr(), ws.numel(),
                                    ops._stream())
    else:
        rc = lib.mmrec_knn_topk_shrink_f32(n, X.data_ptr(), F, F, m, rp, k, norms.data_ptr(), shrink, idx.data_ptr(),
                                           val.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream())
    ops.check(rc, "knn_topk")
    torch.cuda.synchronize()
    r.fallback = lib.mmrec_debug_knn_fallback_rows()
    r.r0 = (m - 1) // r.rows_blk * r.rows_blk
    r.nb = m - r.r0
    r.hdr = _region(ws, o0, off_hdr, 1024, torch.int32)
    r.xpk = _region(ws, o0, off_xpk, r.n_it * FS.TILE * r.KP * 2, torch.int16)
    r.rnorm = _region(ws, o0, off_rnorm, n * 4, torch.float32)
    r.qpk = _region(ws, o0, off_qpk, r.rows_pad * r.KP * 2, torch.int16)
    r.gmax = _region(ws, o0, off_gmax, r.rows_blk * r.G * 4, torch.float32).view(r.rows_blk, r.G)
    r.thr = _region(ws, o0, off_thr, r.rows_blk * 4, torch.float32)
    r.flags = _region(ws, o0, off_flags, r.rows_blk * 4, torch.int32)
    return r


def _f32(bits):
    """The float of a non-negative fp32 bit pattern."""
    return torch.tensor([int(bits)], dtype=torch.int32).view(torch.float32).item()


def knn_check_stages(r, X, rows, k, norms=None, shrink=0.0):
    dev = X.device
    n, F = X.shape
    KP, G, Gv, nb = r.KP, r.G, r.G_valid, r.nb
    qrows = (torch.arange(n, device=dev) if rows is None else rows)[r.r0:]
    hdr = r.hdr.cpu().to(torch.int64) & 0xFFFFFFFF
    assert hdr[0].item() == FS.absmax_bits(X).max().item(), "largest |element|"
    e = FS.fp16_scale_exp(hdr[0:1]).item()
    sc = 2.0 ** e
    up = 1 + (F // 32 + 10) * 2.0 ** -23
    nt = X.double().norm(dim=1)
    rn = r.rnorm.double()
    assert torch.all(rn >= nt) and torch.all(rn <= nt * up), "row norms"
    assert hdr[1].item() == (r.rnorm.view(torch.int32).to(torch.int64)).max().item(), "largest row norm"
    assert torch.equal(r.xpk, FS.pack_tiles(X, torch.tensor([e]), KP, r.n_it * FS.TILE)), "table pack"
    assert torch.equal(r.qpk, FS.pack_tiles(X[qrows], torch.tensor([e]), KP, r.rows_pad)), "query pack"
    assert torch.all(r.gmax[nb:].view(torch.uint8) == SENT) and torch.all(r.thr[nb:].view(torch.uint8) == SENT), \
        "padded query rows were written"
    gmax = r.gmax[:nb]
    S = KP // 16
    A = FS.unpack_tiles(r.qpk, nb, KP).double()
    Xh = FS.unpack_tiles(r.xpk, n, KP).double()
    npad = r.n_it * FS.TILE - n
    mn = _f32(hdr[1])
    un = rn[qrows]
    if norms is not None:
        Rmax, nmin, nmax = _f32(hdr[2]), _f32(0x7FFFFFFF - hdr[3].item()), _f32(hdr[5])
        assert hdr[4].item() == 0
        nq_all = norms[qrows].double()
        bound = torch.tensor([FS.knn_shrink_e(un[i].item(), nq_all[i].item(), mn, Rmax, nmin, nmax, shrink, F, sc)
                              for i in range(nb)], dtype=torch.float64, device=dev)
    else:
        bound = FS.knn_eps_prime(un * sc, mn * sc, F, sc)
    for c0, c1 in _chunks(nb, r.n_it * FS.TILE):
        gk = gmax[c0:c1].double()
        assert torch.all(gk[:, Gv:] == -float("inf")), "groups past the last item must be -inf"
        s = X[qrows[c0:c1]].double() @ X.double().T
        if norms is None:
            dot = A[c0:c1] @ Xh.T
            absd = A[c0:c1].abs() @ Xh.abs().T
            gm = torch.nn.functional.pad(dot, (0, npad), value=-float("inf")).view(c1 - c0, G, 16).amax(-1)[:, :Gv]
            ga = torch.nn.functional.pad(absd, (0, npad)).view(c1 - c0, G, 16).amax(-1)[:, :Gv]
            err = (gk[:, :Gv] - gm).abs()
            assert torch.all(err <= FS.acc_bound(S, ga)), \
                f"pass: group maxima outside the accumulation term, worst {float((err / FS.acc_bound(S, ga)).max()):.3g}"
            v = s * sc * sc
        else:
            D = (norms[qrows[c0:c1], None] * norms[None, :]) + torch.tensor(shrink, dtype=torch.float32, device=dev)
            v = s / D.double()
        gv = torch.nn.functional.pad(v, (0, npad), value=-float("inf")).view(c1 - c0, G, 16).amax(-1)[:, :Gv]
        bad = (gk[:, :Gv] - gv).abs() > bound[c0:c1, None]
        assert not bad.any(), f"pass: {int(bad.sum())} group maxima outside the documented bound of the exact value"
    # threshold
    flags = r.flags[:nb]
    thr = r.thr[:nb].double()
    if k > Gv:
        assert torch.all(flags == 1) and torch.all(torch.isinf(thr))
        return
    assert torch.all(flags == 0), "flags"
    t, kth = FS.rule_threshold(gmax[:, :Gv], torch.full((nb,), k, device=dev), FS.KN_THR_BITS)
    assert torch.all((gmax[:, :Gv] >= t[:, None]).sum(1) >= k) and torch.all(t <= kth)
    t64 = t.double()
    lo = 2 * bound * (1 - 2.0 ** -12) if norms is not None else 2 * bound
    assert torch.all(thr <= t64 - lo), "thr above t - 2 eps'"
    assert torch.all(thr >= t64 - 3 * bound * (1 + 2.0 ** -8)), "thr below t - 3 eps': the margin is vacuous"
    implied = (gmax[:, :Gv].double() >= (thr + lo)[:, None]).sum(1)
    assert torch.all(implied >= k), "fewer than k maxima at or above thr + 2 eps'"


KNN_CASES = [
    # n, F, m (None = all rows), k
    (120, 200, None, 5),
    (120, 200, None, 10),          # k > G_valid = 8: every row flag 1
    (7000, 384, 300, 10),
    (7000, 4096, None, 10),
    (7000, 4100, 1000, 50),        # K tail: the last 64-wide chunk holds 4 real columns
    (7000, 200, 257, 1),
    (23000, 8192, 513, 10),        # 128 chunks through the 4-stage ring
]


@pytest.mark.parametrize("n,F,m,k", KNN_CASES)
def test_knn_stages(dev, n, F, m, k):
    g = torch.Generator(device="cuda").manual_seed(n + F + k)
    X = torch.randn(n, F, generator=g, device=dev)
    X = X / X.norm(dim=1, keepdim=True)
    rows = None if m is None else torch.randperm(n, generator=g, device=dev)[:m]
    r = knn_run(X, rows, k)
    knn_check_stages(r, X, rows, k)


@pytest.mark.parametrize("shrink", [0.0, 10.0, 1e4])
def test_knn_shrink_stages(dev, shrink):
    n, F, m, k = 7000, 384, 300, 10
    g = torch.Generator(device="cuda").manual_seed(5)
    X = torch.randn(n, F, generator=g, device=dev).abs() * torch.rand(n, 1, generator=g, device=dev)
    norms = X.norm(dim=1)
    rows = torch.randperm(n, generator=g, device=dev)[:m]
    r = knn_run(X, rows, k, norms, shrink)
    knn_check_stages(r, X, rows, k, norms, shrink)


# ================================================================================================ accumulation
FAMS = ("big + sub-ulp", "one step", "cancellation", "exponent spread")


def _report(what, a, b, gk, S):
    """Per family: the worst |s~ - a.b| / (S STEP_ERR (1 + 2^-9) sum |a_k b_k|), the summed bound; and for the one-step
    family (every other step zero, so c = 0 where it adds) the worst |s~ - a.b| / (STEP_ERR sum |p|), the assumption of
    a single step itself.  Both must stay <= 1."""
    ex = a.double() @ b.double().T
    ab = a.double().abs() @ b.double().abs().T
    err = (gk.double() - ex).abs()
    ratio = err / FS.acc_bound(S, ab)
    fam = torch.arange(a.shape[0], device=a.device) % 4
    worst = {FAMS[f]: float(ratio[fam == f].max()) for f in range(4)}
    step1 = float((err / (FS.STEP_ERR * ab))[fam == 1].max())
    print(f"\naccumulation {what} (S = {S}): worst ratio to the bound " +
          ", ".join(f"{kk} {v:.4f}" for kk, v in worst.items()) + f"; one step against STEP_ERR sum|p|: {step1:.4f}")
    assert max(worst.values()) <= 1.0, f"{what}: the accumulation bound fails: {worst}"
    assert step1 <= 1.0, f"{what}: one MMA step errs by {step1:.3f} x STEP_ERR sum |p|"
    return worst


def _probe_rows(R, K, seed, dev):
    fam = torch.arange(R) % 4
    rows = torch.zeros(R, K)
    for f in range(4):
        rows[fam == f] = FS.probe_rows(int((fam == f).sum()), K, seed + f, f)
    return rows.to(dev)


@pytest.mark.parametrize("d", [32, 64, 128])
def test_cf_accumulation_probes(dev, d):
    """K3: one probe item per group of 16 (the rest zero rows, which score exactly 0), positive probe scores: every group
    maximum is one probe's s~."""
    I, B = 7000, 256
    Gp = -(-I // 16)
    a = _probe_rows(B, d, 100 + d, dev)
    b = FS.probe_items(Gp, d, seed=d).to(dev)
    pos = torch.clamp(torch.arange(Gp) * 16 + torch.arange(Gp) % 16, max=I - 1).to(dev)
    ie = torch.zeros(I, d, device=dev)
    ie[pos] = b
    r = cf_run(a, ie, None, None, 1, in_call=True)
    assert r.KP == d
    _report(f"K3 KP={d}", a, b, r.gmax[:B, :Gp], d // 16)


@pytest.mark.parametrize("F", [200, 384, 4096, 8192])
def test_knn_accumulation_probes(dev, F):
    """K7: the probe queries are table rows 0 .. 255, queried through rows=; one probe item per later group of 16."""
    Q, Gp = 256, 300
    K = F // 16 * 16
    a = torch.zeros(Q, F, device=dev)
    a[:, :K] = _probe_rows(Q, K, 200 + F, dev)
    b = torch.zeros(Gp, F, device=dev)
    b[:, :K] = FS.probe_items(Gp, K, seed=F).to(dev)
    n = Q + 16 * Gp
    X = torch.zeros(n, F, device=dev)
    X[:Q] = a
    pos = Q + torch.arange(Gp, device=dev) * 16 + torch.arange(Gp, device=dev) % 16
    X[pos] = b
    r = knn_run(X, torch.arange(Q, device=dev), 1)
    assert r.KP // 16 == FS.knn_steps(F)
    _report(f"K7 F={F}", a, b, r.gmax[:Q, Q // 16:Q // 16 + Gp], r.KP // 16)


def _report_worst(what, a, lab, x, b, gk):
    """Worst-case probes (filter_stages.worst_rows): per label and per guard level g = 5 - e (the small products just
    below 2^(5 - g) next to P = 2^28), the worst |s~ - a.b| / (2^-22 (|c| + sum |p|)) of the one step that adds them.
    Every other step adds exact zeros, so that is the error of that step; it must stay within STEP_ERR."""
    ex = a.double() @ b.double().T
    ab = a.double().abs() @ b.double().abs().T                # = |c| + sum |p| of the step (c = P or 0)
    ratio = (gk.double() - ex).abs() / (2.0 ** -22 * ab)
    y = torch.arange(b.shape[0], device=a.device) % 4
    g = 5 - (x.to(a.device)[:, None] + y[None, :] + 1)
    lab = lab.to(a.device)
    lines = []
    for lv in range(4):
        per = [float(ratio[(lab[:, None] == t) & (g == lv)].max()) for t in range(4)]
        lines.append(f"g={lv}: " + ", ".join(f"{n} {v:.3f}" for n, v in zip(FS.WORST, per)))
    worst = float(ratio.max())
    print(f"\nworst-case step {what}: max {worst:.4f} x 2^-22\n  " + "\n  ".join(lines))
    assert worst <= FS.STEP_ERR / 2.0 ** -22, f"{what}: one MMA step errs by {worst:.3f} x 2^-22 (|c| + sum |p|)"


@pytest.mark.parametrize("d", [32, 128])
def test_cf_worst_step_probes(dev, d):
    """K3, as test_cf_accumulation_probes, with the worst-case operands."""
    I, B = 7000, 256
    Gp = -(-I // 16)
    a, lab, x = FS.worst_rows(B, d)
    a = a.to(dev)
    b = FS.worst_items(Gp, d).to(dev)
    pos = torch.clamp(torch.arange(Gp) * 16 + torch.arange(Gp) % 16, max=I - 1).to(dev)
    ie = torch.zeros(I, d, device=dev)
    ie[pos] = b
    r = cf_run(a, ie, None, None, 1, in_call=True)
    _report_worst(f"K3 KP={d}", a, lab, x, b, r.gmax[:B, :Gp])


@pytest.mark.parametrize("F", [384, 4096])
def test_knn_worst_step_probes(dev, F):
    """K7, as test_knn_accumulation_probes, with the worst-case operands."""
    Q, Gp = 256, 300
    a, lab, x = FS.worst_rows(Q, F)
    a = a.to(dev)
    b = FS.worst_items(Gp, F).to(dev)
    n = Q + 16 * Gp
    X = torch.zeros(n, F, device=dev)
    X[:Q] = a
    pos = Q + torch.arange(Gp, device=dev) * 16 + torch.arange(Gp, device=dev) % 16
    X[pos] = b
    r = knn_run(X, torch.arange(Q, device=dev), 1)
    _report_worst(f"K7 F={F}", a, lab, x, b, r.gmax[:Q, Q // 16:Q // 16 + Gp])
