"""CPU restatement of ItemKNNCBF (src/models/itemknncbf.py) with the same torch ops in the same order, the ordered sparse
sums K9 promises, and a host emulation of K9's sparse ranking rule (csrc/sparse_score.cu).  Test infrastructure: the
product never imports it."""
import numpy as np
import torch


def item_sim_topk(features: torch.Tensor, knn_k: int, shrink):
    """`build_item_sim_matrix` (itemknncbf.py:56-65) up to its top-k: (values [I, k], indices [I, k]) before the scatter."""
    i_norm = torch.norm(features, p=2, dim=-1, keepdim=True)
    ij_norm = i_norm * i_norm.T + shrink
    ij = torch.mm(features, features.T)
    sim = ij.div(ij_norm)
    return torch.topk(sim, knn_k, dim=-1)


def item_sim_topk_f64(features: torch.Tensor, knn_k: int, shrink):
    """The same similarity evaluated in float64 and rounded once to float32: a value that does not depend on the CPU's
    fp32 GEMM code path (which changes the low bits of `item_sim_topk` from one instruction set to another).  Ranked on the
    float64 values, equal values by ascending index.  Returns (values fp32 [I, k], indices [I, k])."""
    x = features.double()
    nrm = torch.norm(x, p=2, dim=-1, keepdim=True)
    sim = (x @ x.T) / (nrm * nrm.T + shrink)
    order = torch.sort(sim, dim=-1, descending=True, stable=True).indices[:, :knn_k]
    return torch.gather(sim, 1, order).float(), order


def sim_error_bound(features: torch.Tensor, shrink):
    """Per pair, a bound on |fp32 similarity - exact| for any fp32 evaluation of `item_sim_topk`'s expression (a dot product
    of F terms in any order, the norms, one multiply, one add, one division): 2 F 2^-24 |x||y| / (|x||y| + shrink) + 2^-22
    |sim|, from the standard bound gamma_F on a sum of F rounded terms."""
    x = features.double()
    F = x.shape[1]
    nrm = torch.norm(x, p=2, dim=-1, keepdim=True)
    nn = nrm * nrm.T
    sim = (x @ x.T) / (nn + shrink)
    return 2 * F * 2.0 ** -24 * nn / (nn + shrink) + 2.0 ** -22 * sim.abs()


def knn_agrees(got_val, got_idx, want_val, want_idx, features, shrink):
    """Two fp32 evaluations of the kNN of `item_sim_topk` agree: the same neighbours per row except where the exact
    similarities of the swapped items lie within both evaluations' error bounds of each other, and every value within
    those bounds of the other's.  Returns (ok, rows that differ in their neighbours)."""
    x = features.double()
    nrm = torch.norm(x, p=2, dim=-1, keepdim=True)
    sim = ((x @ x.T) / (nrm * nrm.T + shrink)).numpy()
    tol = 2 * sim_error_bound(features, shrink).numpy()
    gv, gi, wv, wi = (np.asarray(a) for a in (got_val, got_idx, want_val, want_idx))
    rows = 0
    for r in range(gi.shape[0]):
        a, b = set(gi[r].tolist()), set(wi[r].tolist())
        if a != b:
            rows += 1
            lo = min(sim[r, j] - tol[r, j] for j in a - b)
            hi = max(sim[r, j] + tol[r, j] for j in b - a)
            if lo > hi:
                return False, rows
        for v, j in zip(gv[r], gi[r]):
            if abs(float(v) - sim[r, j]) > tol[r, j]:
                return False, rows
        for v, j in zip(wv[r], wi[r]):
            if abs(float(v) - sim[r, j]) > tol[r, j]:
                return False, rows
    return True, rows


def features(v_feat, t_feat):
    """itemknncbf.py:43-48: cat(v, t), else the one modality present."""
    if v_feat is not None and t_feat is not None:
        return torch.cat((v_feat, t_feat), -1)
    return v_feat if v_feat is not None else t_feat


def ordered_scores(inter_row, inter_col, inter_val, n_users, knn_val, knn_ind, order="ascending", users=None):
    """score[u, j] = sum over the entries of R(u) of r * S[i, j] in fp32, one rounding per entry, from +0.0.

    order = "ascending": R's entries of a row in ascending column order (K9's contract); "stored": in the order they are
    given.  Each step is fl(fl(r * s) + acc), equal to fmaf(r, s, acc) whenever r * s is exact in fp32 (r = 1 always)."""
    inter_row, inter_col = np.asarray(inter_row, np.int64), np.asarray(inter_col, np.int64)
    inter_val = np.asarray(inter_val, np.float32)
    knn_val, knn_ind = np.asarray(knn_val, np.float32), np.asarray(knn_ind, np.int64)
    n_items = knn_val.shape[0]
    perm = np.lexsort((inter_col, inter_row)) if order == "ascending" else np.argsort(inter_row, kind="stable")
    users = np.arange(n_users) if users is None else np.asarray(users, np.int64)
    out = np.zeros((len(users), n_items), np.float32)
    by_user = {}
    for p in perm:
        by_user.setdefault(int(inter_row[p]), []).append(p)
    for b, u in enumerate(users):
        acc = out[b]
        for p in by_user.get(int(u), []):
            i, r = inter_col[p], inter_val[p]
            cols = knn_ind[i]
            acc[cols] = (np.float32(r) * knn_val[i]).astype(np.float32) + acc[cols]
    return out


def float_key(v):
    """csrc/common.cuh's order-preserving key: -0.0 below +0.0, positive NaN largest."""
    u = np.asarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000).astype(np.uint64)


def dense_rank(row, masked, k):
    """`row[masked] = -1e10` then the top k, values descending by float_key, equal values by ascending index
    (mmrec_mask_f32 + mmrec_topk_rows_f32)."""
    row = np.array(row, np.float32)
    m = np.asarray(masked, np.int64)
    row[m[(m >= 0) & (m < len(row))]] = np.float32(-1e10)
    order = np.lexsort((np.arange(len(row)), -float_key(row).astype(np.int64)))[:k]
    return row[order], order


def sparse_rank(cols, sums, masked, n_items, k):
    """K9's ranking rule from the summed columns alone (csrc/sparse_score.cu, step 5): the exceptions -- masked items
    (-1e10) and unmasked columns whose sum is not +0.0 -- sorted on (float_key desc, index asc); the output is the
    exceptions above +0.0, then every other item (+0.0) in ascending index, then the remaining exceptions."""
    cols, sums = np.asarray(cols, np.int64), np.asarray(sums, np.float32)
    m = np.unique(np.asarray(masked, np.int64))
    m = m[(m >= 0) & (m < n_items)]
    keep = ~np.isin(cols, m) & (sums.view(np.uint32) != 0)
    ex_idx = np.concatenate([m, cols[keep]])
    ex_val = np.concatenate([np.full(len(m), -1e10, np.float32), sums[keep]])
    order = np.lexsort((ex_idx, -float_key(ex_val).astype(np.int64)))
    ex_idx, ex_val = ex_idx[order], ex_val[order]
    A = int((float_key(ex_val) > 0x80000000).sum())
    zero = np.setdiff1d(np.arange(n_items), ex_idx)
    idx = np.concatenate([ex_idx[:A], zero, ex_idx[A:]])[:k]
    val = np.concatenate([ex_val[:A], np.zeros(len(zero), np.float32), ex_val[A:]])[:k]
    return val, idx
