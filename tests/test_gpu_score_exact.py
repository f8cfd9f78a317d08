"""The fused score + mask + top-k (K3, csrc/score_cf.cu) against its contract, bit for bit: whichever kernel serves a
row (cf_final_kernel after the certified fp16 filter, or cf_exact_kernel), the row is the exact fp32 top-k of the chain
arithmetic documented in that file, ordered by float_key, equal values -> lower item index.  The reference is
oracle.mmrec_oracle.cf_exact_topk (its emulation of the arithmetic is checked in tests/test_fp32_chain_host.py).

Every case compares indices and value BITS with zero tolerance, runs both the forced "fused" path and "auto", with and
without a packed Catalog, and asserts how many rows of the last row block the exact kernel took
(ops.fused_fallback_rows): that is how each test names the branch it reaches."""
import math

import pytest
import torch

from oracle import mmrec_oracle as O

pytestmark = pytest.mark.gpu

# shape rules of score_cf.cu, restated to name the branch a case takes
CF_TILE = 128


def cf_gw(n_items):
    return 1 if n_items <= 16384 else (2 if n_items <= 32768 else (4 if n_items <= 65536 else 8))


def cf_groups(n_items):
    """(G, G_valid): group maxima per row, and those holding at least one real item."""
    n_it = -(-n_items // CF_TILE)
    return n_it * (8 // cf_gw(n_items)), -(-n_items // (16 * cf_gw(n_items)))


def cf_rows_blk(B, n_items):
    n_it = -(-n_items // CF_TILE)
    G = cf_groups(n_items)[0]
    rb = (512 << 20) // (G * 4 + n_it * 16) // (2 * CF_TILE) * (2 * CF_TILE)
    return min(B, min(max(rb, 2 * CF_TILE), 65536))


def need_rows(mask, B, k, G_valid):
    """Rows whose need = k + (mask entries of the row, duplicates and other shards' columns included) exceeds the
    groups: cf_thr_kernel sends them to the exact kernel."""
    if mask is None:
        return 0
    r = mask[0][(mask[0] >= 0) & (mask[0] < B)]
    cnt = torch.bincount(r.cpu(), minlength=B)
    return int((k + cnt > G_valid).sum())


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    from mmrec_b200 import _lib
    _lib.require_device()
    return torch.device("cuda:0")


def bits(v):
    return v.detach().cpu().contiguous().view(torch.int32)


def assert_same(val, idx, rv, ri, what=""):
    val, idx = val.cpu(), idx.cpu()
    bad = (idx != ri).any(dim=1) | (bits(val) != bits(rv)).any(dim=1)
    if bad.any():
        r = int(torch.nonzero(bad)[0])
        c = int(torch.nonzero((idx[r] != ri[r]) | (bits(val[r]) != bits(rv[r])))[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {len(bad)} rows differ from the exact fp32 top-k; first row {r} "
                             f"from rank {c}: got {idx[r, c:c + 4].tolist()} {val[r, c:c + 4].tolist()}, want "
                             f"{ri[r, c:c + 4].tolist()} {rv[r, c:c + 4].tolist()}")


def fused(ue, ie, users, mask, k, item_offset=0):
    """ops.score_topk forced to "fused" and through "auto", with and without a Catalog: all four must agree bit for
    bit, and on the rows the exact kernel took.  Returns (values, indices, fallback rows of the last row block)."""
    from mmrec_b200 import ops
    res = []
    try:
        for path in ("fused", "auto"):
            ops.set_score_path(path)
            v, i = ops.score_topk(ue, ie, users, mask, k, item_offset)
            res.append((v, i, ops.fused_fallback_rows()))
            if path == "fused":
                cat = ops.Catalog(ie)
                v, i = ops.score_topk(ue, cat.item_e, users, mask, k, item_offset, catalog=cat)
                res.append((v, i, ops.fused_fallback_rows()))
                del cat
    finally:
        ops.set_score_path("auto")
    v0, i0, f0 = res[0]
    for v, i, f in res[1:]:
        assert torch.equal(i, i0) and torch.equal(bits(v), bits(v0)) and f == f0
    return v0, i0, f0


def check(ue, ie, users, mask, k, item_offset=0, fallback=0, what=""):
    """The fused result equals cf_exact_topk; `fallback` = expected exact-kernel rows (int, or a predicate)."""
    v, i, fb = fused(ue, ie, users, mask, k, item_offset)
    rv, ri = O.cf_exact_topk(ue, ie, users, mask, k, item_offset, device=ue.device)
    assert_same(v, i, rv, ri, what)
    if callable(fallback):
        assert fallback(fb), f"{what}: {fb} rows took the exact kernel"
    else:
        assert fb == fallback, f"{what}: {fb} rows took the exact kernel, expected {fallback}"
    return v, i, fb


def rand_case(dev, B, U, I, d, seed, scale=0.1, per_row=6, off=0):
    g = torch.Generator().manual_seed(seed)
    ue = torch.randn(U, d, generator=g) * scale
    ie = torch.randn(I, d, generator=g) * scale
    users = torch.randint(0, U, (B,), generator=g)
    nm = B * per_row
    mask = torch.stack([torch.randint(0, B, (nm,), generator=g), torch.randint(0, I, (nm,), generator=g) + off])
    return ue.to(dev), ie.to(dev), users.to(dev), mask.to(dev), g


# ------------------------------------------------------------------------------------------------ widths, layouts
@pytest.mark.parametrize("d", [1, 3, 31, 32, 33, 63, 64, 65, 100, 127, 128])
def test_exact_widths(dev, d):
    """L = 8 / 16 / 32 blocks (d <= 32 / 64 / 128); d % 4 != 0 takes the scalar loads in both exact-score kernels."""
    ue, ie, users, mask, _ = rand_case(dev, 300, 400, 3000, d, seed=d)
    check(ue, ie, users, mask, 20, what=f"d={d}")


def test_exact_misaligned_and_strided(dev):
    """Item / user tables not 16-byte aligned, and leading dimensions > d (through the C ABI: ops always passes
    contiguous tensors): the scalar-load paths, and the vector path with a row stride."""
    from mmrec_b200 import _lib, ops
    B, U, I, d, k = 300, 400, 3000, 64, 20
    ue, ie, users, mask, _ = rand_case(dev, B, U, I, d, seed=7)
    rv, ri = O.cf_exact_topk(ue, ie, users, mask, k, device=dev)
    ie_m = torch.empty(I * d + 1, device=dev)[1:].view(I, d); ie_m.copy_(ie)
    ue_m = torch.empty(U * d + 1, device=dev)[1:].view(U, d); ue_m.copy_(ue)
    assert ie_m.data_ptr() % 16 == 4 and ue_m.data_ptr() % 16 == 4
    for a, b in [(ue, ie_m), (ue_m, ie), (ue_m, ie_m)]:
        v, i, fb = fused(a, b, users, mask, k)
        assert_same(v, i, rv, ri, "misaligned")
        assert fb == 0
    lib = _lib.load()
    nnz = mask.shape[1]
    for ldu, ldi in [(d + 5, d), (d, d + 3), (d + 4, d + 4), (d + 1, d + 8)]:
        ub = torch.zeros(U, ldu, device=dev); ub[:, :d] = ue
        ib = torch.zeros(I, ldi, device=dev); ib[:, :d] = ie
        for with_cat in (False, True):
            ws = torch.empty(lib.mmrec_score_topk_workspace_bytes(B, I, d, k) + 4 * nnz + 4096, dtype=torch.uint8, device=dev)
            idx = torch.empty(B, k, dtype=torch.int64, device=dev); val = torch.empty(B, k, device=dev)
            cat_ptr, cat = None, None
            if with_cat:
                nbytes = lib.mmrec_catalog_bytes(I, d)
                cat = torch.empty(nbytes + 1024, dtype=torch.uint8, device=dev)
                cat_ptr = (cat.data_ptr() + 1023) // 1024 * 1024
                ops.check(lib.mmrec_catalog_pack_f32(I, ib.data_ptr(), ldi, d, cat_ptr, nbytes, ops._stream()), "catalog_pack")
            ops.check(lib.mmrec_score_topk_cat_f32(B, users.data_ptr(), ub.data_ptr(), ldu, I, ib.data_ptr(), ldi, d, cat_ptr, nnz,
                                                   mask[0].contiguous().data_ptr(), mask[1].contiguous().data_ptr(), k, 0,
                                                   idx.data_ptr(), val.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream()),
                      "score_topk_cat")
            assert lib.mmrec_debug_fused_fallback_rows(ws.data_ptr(), B, I, d, k, nnz, int(not with_cat)) == 0
            assert_same(val, idx, rv, ri, f"ldu={ldu} ldi={ldi} cat={with_cat}")


# ------------------------------------------------------------------------------------------------ k and group counts
@pytest.mark.parametrize("k", [1, 50, 100, 256])
def test_exact_k_and_group_boundary(dev, k):
    """The smallest catalogue with G >= 2k (G == 2k exactly where 8 | 2k) is fused; one item tile less is not
    (fallback -1: the unfused tensor-core path, equal to ops.score + ops.mask_topk).  k > 128 ranks in several sweeps."""
    from mmrec_b200 import ops
    n_min = max(1, -(-2 * k // 8))                                   # item tiles for G = 8 n_it >= 2k
    I = 128 * (n_min - 1) + 1 if n_min > 1 else 129
    G, G_valid = cf_groups(I)
    assert G >= 2 * k and (2 * k % 8 or G == 2 * k)
    B = 300
    ue, ie, users, mask, _ = rand_case(dev, B, 400, I, 64, seed=k, per_row=2)
    check(ue, ie, users, mask, k, fallback=need_rows(mask, B, k, G_valid), what=f"k={k} I={I}")
    if n_min > 1:
        I2 = 128 * (n_min - 1)
        assert cf_groups(I2)[0] < 2 * k
        ie2 = ie[:I2].contiguous()
        mask2 = mask[:, mask[1] < I2]
        v, i, fb = fused(ue, ie2, users, mask2, k)
        assert fb == -1
        S = ops.score(ue, ie2, users)
        v2, i2 = ops.mask_topk(S, mask2, k)
        assert torch.equal(i, i2) and torch.equal(bits(v), bits(v2))


@pytest.mark.parametrize("I", [8191, 8192, 8193, 16384, 16385, 32768, 32769, 65536, 65537, 131072, 131073])
def test_exact_item_counts(dev, I):
    """Group width gw = 1 / 2 / 4 / 8 items-per-16 switches at 16 384 / 32 768 / 65 536 items, the threshold search at
    G = 512 (coarse, 16 keys per lane) / 1024 (coarse, 32) / beyond (radix), ragged last item tiles (I % 128 = 127, 0, 1)."""
    G, G_valid = cf_groups(I)
    ue, ie, users, mask, _ = rand_case(dev, 257, 300, I, 64, seed=I, per_row=4)
    check(ue, ie, users, mask, 50, fallback=need_rows(mask, 257, 50, G_valid), what=f"I={I} G={G} gw={cf_gw(I)}")


# ------------------------------------------------------------------------------------------------ batch sizes, row blocks
@pytest.mark.parametrize("B", [1, 255, 256, 257, 4097, 9000])
def test_exact_batch_sizes(dev, B):
    """Ragged user-tile pairs; B = 9000 > 8192 builds the mask CSR on the large-mask route (count, scan, fill)."""
    I, k = 3000, 20
    ue, ie, users, mask, g = rand_case(dev, B, max(B, 300), I, 32, seed=B)
    mask = torch.cat([mask, torch.tensor([[-1, B, B + 3], [5, 6, 7]], device=dev)], 1)     # rows outside the batch
    check(ue, ie, users, mask, k, fallback=need_rows(mask, B, k, cf_groups(I)[1]), what=f"B={B}")


def test_exact_large_mask(dev):
    """B = 4096 with more than 2^18 mask entries: the large-mask route at a batch the small route would take."""
    B, I, k = 4096, 3000, 20
    ue, ie, users, mask, g = rand_case(dev, B, 5000, I, 32, seed=3, per_row=70)
    assert mask.shape[1] > (1 << 18)
    check(ue, ie, users, mask, k, fallback=need_rows(mask, B, k, cf_groups(I)[1]), what="large mask")


@pytest.mark.parametrize("with_users", [False, True])
def test_exact_two_row_blocks(dev, with_users):
    """1 000 003 items, d = 32, B = 4096 (an unsharded evaluation batch of the largest configuration): the group maxima
    + bitmap exceed 512 MB, so the batch runs as two row blocks (the users / Ue / mask-pointer / output offsets)."""
    B, I, d, k = 4096, 1_000_003, 32, 50
    assert cf_rows_blk(B, I) < B
    ue, ie, users, mask, _ = rand_case(dev, B, 5000 if with_users else B, I, d, seed=11, per_row=10)
    check(ue, ie, users if with_users else None, mask, k, what="two row blocks")


# ------------------------------------------------------------------------------------------------ masks
def test_exact_masks(dev):
    """Unsorted mask with duplicates and rows outside the batch (== the same mask sorted); need == G_valid (served)
    and need == G_valid + 1 (exact kernel); a row with fewer than k unmasked items (masked ones fill in at -1e10)."""
    B, U, I, d, k = 300, 400, 800, 48, 20       # few items: at need == G_valid the threshold is the lowest group
    G, G_valid = cf_groups(I)                   # maximum, and ~1/4 of the catalogue stays below the 512-candidate cap
    g = torch.Generator().manual_seed(21)
    ue = (torch.randn(U, d, generator=g) * 0.1).to(dev); ie = (torch.randn(I, d, generator=g) * 0.1).to(dev)
    users = torch.randint(0, U, (B,), generator=g).to(dev)
    r = torch.randint(3, B, (B * 5,), generator=g); c = torch.randint(0, I, (B * 5,), generator=g)
    rows = [r, r[:200], torch.tensor([-1, -5, B, B + 1])]
    cols = [c, c[:200], torch.tensor([1, 2, 3, 4])]
    for row, n in [(0, G_valid - k), (1, G_valid - k + 1), (2, I - k + 5)]:
        rows.append(torch.full((n,), row)); cols.append(torch.randperm(I, generator=g)[:n])
    mask = torch.stack([torch.cat(rows), torch.cat(cols)])
    mask = mask[:, torch.randperm(mask.shape[1], generator=g)].to(dev)
    assert need_rows(mask, B, k, G_valid) == 2                       # rows 1 and 2
    v, i, _ = check(ue, ie, users, mask, k, fallback=2, what="unsorted mask")
    assert torch.all(v[2, k - 5:].cpu() == O.MASKED_SCORE)
    srt = mask[:, torch.argsort(mask[0], stable=True)]
    v2, i2, fb = fused(ue, ie, users, srt, k)
    assert torch.equal(i, i2) and torch.equal(bits(v), bits(v2)) and fb == 2
    # a shard: global columns, some of them in other shards (ignored, but counted in need)
    off = 1000
    ms = torch.stack([r, c + off - 40]).to(dev)
    check(ue, ie, users, ms, k, item_offset=off, fallback=need_rows(ms, B, k, G_valid), what="item_offset")


@pytest.mark.parametrize("route", ["sorted", "unsorted", "large"])
def test_mask_columns_wrapping_32_bits(dev, route):
    """Mask columns item_offset + 2^32 + j and item_offset - 2^32 + j lie outside the shard, so ops.mask_topk ignores
    them, although their low 32 bits name item j -- here the first and second of the row's unmasked top-k.  The fused
    call must ignore them too (they still count in need), whichever route builds the mask CSR: rows in order, out of
    order, or B > 8192.  Quantised values: the unfused scores are exact, the same bits as the fused chain."""
    from mmrec_b200 import ops
    B = 9000 if route == "large" else 300
    I, d, k, off = 3000, 32, 20, 1000
    g = torch.Generator().manual_seed(41)
    ue = (torch.randint(-16, 17, (B, d), generator=g).float() / 64).to(dev)
    ie = (torch.randint(-16, 17, (I, d), generator=g).float() / 64).to(dev)
    mask = torch.stack([torch.randint(0, B, (B * 4,), generator=g), torch.randint(0, I, (B * 4,), generator=g) + off]).to(dev)
    _, top = ops.mask_topk(ops.score(ue, ie), mask, 2, off)
    wrap = torch.stack([torch.arange(B, device=dev).repeat(2), torch.cat([top[:, 0] + 2 ** 32, top[:, 1] - 2 ** 32])])
    m = torch.cat([mask, wrap], 1)
    order = torch.randperm(m.shape[1], generator=g) if route == "unsorted" else torch.argsort(m[0].cpu(), stable=True)
    m = m[:, order.to(dev)]
    v, i, _ = check(ue, ie, None, m, k, item_offset=off, fallback=lambda fb: fb <= B // 8, what=route)
    rv, ri = ops.mask_topk(ops.score(ue, ie), m, k, off)
    assert torch.equal(i, ri) and torch.equal(bits(v), bits(rv))


# ------------------------------------------------------------------------------------------------ adversarial values
def test_exact_quantised_ties(dev):
    """Multiples of 2^-6: exact scores and exact ties at the k boundary, ranked by the tie pass of cf_final_kernel."""
    B, I, d, k = 256, 4000, 32, 50
    g = torch.Generator().manual_seed(5)
    ue = torch.randint(-4, 5, (B, d), generator=g).float() / 64; ie = torch.randint(-4, 5, (I, d), generator=g).float() / 64
    mask = torch.stack([torch.randint(0, B, (B * 4,), generator=g), torch.randint(0, I, (B * 4,), generator=g)])
    v, i, _ = check(ue.to(dev), ie.to(dev), None, mask.to(dev), k, what="quantised")
    s = ue.double() @ ie.double().T
    s[mask[0], mask[1]] = -1e10
    kth = v[:, k - 1].cpu().double()
    tied_out = (s == kth[:, None]).sum(1) > (v.cpu().double() == kth[:, None]).sum(1)
    assert tied_out.float().mean().item() > 0.25                     # the boundary really is a tie in many rows


def cluster(I, d, rel, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(d, generator=g)
    return base + torch.randn(I, d, generator=g) * (rel * base.norm().item() / math.sqrt(d)), g


def test_exact_tight_cluster(dev):
    """A catalogue of one tight cluster, 140 000 items (G > 1024: the radix threshold search).  At 2^-5 relative spread
    the filter keeps a few hundred candidates per row and still serves every row; at 2^-10 nothing separates within the
    certified margin, every row exceeds 512 candidates and the exact kernel serves it."""
    B, I, d, k = 256, 140_000, 64, 50
    for rel, fb in [(2.0 ** -4, 0), (2.0 ** -10, B)]:
        ie, g = cluster(I, d, rel, seed=9)
        ue = torch.randn(B, d, generator=g)
        check(ue.to(dev), ie.to(dev), None, None, k, fallback=fb, what=f"cluster {rel}")


def test_exact_condemned_rows(dev):
    """More than 512 near-duplicates at the top of one row (condemn(4)), a zero user row (every item ties at +0, all
    candidates), a user row holding +inf (non-finite flag): exactly those rows take the exact kernel."""
    B, I, d, k = 64, 3000, 32, 20
    g = torch.Generator().manual_seed(13)
    ue = torch.randn(B, d, generator=g); ie = torch.randn(I, d, generator=g)
    ue[:, 0] = 0.0
    ie[:600] = torch.randn(600, d, generator=g) * 1e-3
    ie[:600, 0] = 10.0 + torch.randn(600, generator=g) * 1e-4
    ue[0] = 0.0; ue[0, 0] = 5.0
    mask = torch.stack([torch.randint(0, B, (B * 3,), generator=g), torch.randint(0, I, (B * 3,), generator=g)])
    check(ue.to(dev), ie.to(dev), None, mask.to(dev), k, fallback=1, what="near-duplicates")
    uz = ue.clone(); uz[0, 1:] = torch.randn(d - 1, generator=g); uz[0, 0] = 0.0; uz[5] = 0.0
    v, i, _ = check(uz.to(dev), ie.to(dev), None, mask.to(dev), k, fallback=1, what="zero row")
    assert torch.all(bits(v[5]) == 0)
    ui = uz.clone(); ui[5, 1:] = torch.randn(d - 1, generator=g); ui[9, 3] = float("inf")
    check(ui.to(dev), ie.to(dev), None, mask.to(dev), k, fallback=1, what="inf row")


def test_exact_nan_item(dev):
    """An item holding +inf: its score is NaN for users with a zero in that column (ranked first: NaN is the largest
    key), +inf or -inf for the others; the catalogue is non-finite, so every row takes the exact kernel."""
    B, I, d, k = 32, 2000, 32, 20
    g = torch.Generator().manual_seed(17)
    ue = torch.randn(B, d, generator=g); ie = torch.randn(I, d, generator=g)
    ie[7, 0] = float("inf")
    ue[:16, 0] = 0.0
    v, i, _ = check(ue.to(dev), ie.to(dev), None, None, k, fallback=B, what="nan item")
    assert torch.all(i[:16, 0].cpu() == 7) and torch.all(bits(v[:16, 0]) == 0x7FFFFFFF)
    pos = ue[:, 0] > 0
    assert torch.all(i[pos, 0].cpu() == 7) and torch.all(torch.isinf(v[pos, 0].cpu()))


@pytest.mark.parametrize("su,si", [(1e-25, 0.1), (0.1, 1e-25), (1e18, 0.1), (1e20, 0.1)])
def test_exact_magnitudes(dev, su, si):
    """Tiny and huge rows.  The filter's row norms are taken after the power-of-two scaling: squares of elements near
    1e-25 would underflow to 0 and zero the certified margin (rows served with true top-k members dropped), squares of
    elements near 1e20 would overflow and send every row to the exact kernel."""
    B, I, d, k = 300, 5000, 64, 50
    ue, ie, users, mask, g = rand_case(dev, B, 300, I, d, seed=23)
    check(ue * (su / 0.1), ie * (si / 0.1), users, mask, k, fallback=need_rows(mask, B, k, cf_groups(I)[1]), what=f"random {su} {si}")
    # a tight cluster: the margin is all that keeps the true top-k (every row exceeds 512 candidates and goes exact)
    ic, g = cluster(I, d, 2.0 ** -10, seed=29)
    uc = torch.randn(64, d, generator=g)
    check((uc * su).to(dev), (ic * si).to(dev), None, None, k, fallback=64, what=f"cluster {su} {si}")


def test_power_of_two_scaling_is_exact(dev):
    """Metamorphic, no emulation: scaling the users or the items by a power of two that keeps every product normal
    leaves the indices identical and scales the values by exactly that power."""
    B, I, d, k = 300, 5000, 64, 50
    ue, ie, users, mask, g = rand_case(dev, B, 300, I, d, seed=31)
    v, i, fb = fused(ue, ie, users, mask, k)
    for a, b, s in [(2.0 ** 40, 1.0, 2.0 ** 40), (1.0, 2.0 ** -30, 2.0 ** -30), (2.0 ** -50, 2.0 ** 20, 2.0 ** -30)]:
        v2, i2, fb2 = fused(ue * a, ie * b, users, mask, k)
        assert torch.equal(i, i2) and fb2 == fb
        assert torch.equal(bits(v2), bits(v * s))
