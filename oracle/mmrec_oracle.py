"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY, NOT PRODUCT CODE.

A restatement, in plain numpy / torch-CPU fp32, of the algorithm on MMRec's hot
path (SURVEY.md section 8a): graph normalisation, per-epoch edge pruning, LightGCN
style sparse propagation, modality projection / fusion, full-catalog scoring and
the trainer's mask + top-k.  Every function cites the reference lines it follows
(paths relative to the root of enoche/MMRec).

Who may import this file: `tests/`, `__graft_entry__.smoke()` and the
`cpu_baseline` / `--impl reference` legs of `bench.py` -- as the checker or the
timed CPU baseline, never as part of what `mmrec_b200` ships.  The product path
(`mmrec_b200.ops`) raises if its CUDA library is missing; it never falls back here.

Where the arithmetic lives: the reference's numerics are PyTorch's (pinned
torch==1.11.0 in `requirements.txt:5`; this container has 2.11.0) -- ATen sparse
COO addmm, `mm`, `topk`.  The restatement therefore calls the same torch CPU ops
in the same order, so on CPU it is bit-identical to the reference.

PARITY PIN: the reference ships no tests / golden vectors (SURVEY.md section 4), so
the oracle is pinned against outputs of the unmodified reference itself, run by
`tests/golden/make_golden.py` and committed as
`tests/golden/*_tiny.npz`; `tests/test_oracle_golden.py` checks every function here
against those files (bit-exact for indices and for values produced by the same
torch ops).  MMGCN: torch_geometric is not a dependency, so its one PyG primitive (`mmgcn_mean_aggregate`) stays
"parity unpinned"; the model code around it is pinned to the reference run under a shim of that primitive
(tests/golden/mmgcn_tiny.npz).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------------------
# a1: normalised user-item adjacency
# --------------------------------------------------------------------------------------


def norm_adj_coo(inter_row, inter_col, n_users, n_items):
    """A_hat = D^-1/2 [[0,R],[R^T,0]] D^-1/2 as un-coalesced torch COO (fp32 values, int64 indices).

    Follows `src/models/freedom.py:102-126` (identical bodies: `bm3.py:58-82`,
    `lightgcn.py:65-101`, `layergcn.py:91-115`, `common/encoders.py:39-75`): binary adjacency,
    degree + 1e-7 in float64, power -0.5, L = (D*A)*D in float64, ONE rounding to fp32
    (`torch.FloatTensor(L.data)`), entries in row-major order with ascending columns.
    """
    r = np.asarray(inter_row, dtype=np.int64)
    c = np.asarray(inter_col, dtype=np.int64)
    n = n_users + n_items
    # the dict of (r, c) keys de-duplicates repeated interactions (freedom.py:107-110)
    key = np.unique(np.concatenate([r * n + (c + n_users), (c + n_users) * n + r]))
    rows, cols = key // n, key % n
    deg = np.bincount(rows, minlength=n).astype(np.float64) + 1e-7       # (A > 0).sum(axis=1) + 1e-7
    with np.errstate(divide="ignore"):
        dinv = np.power(deg, -0.5)                                        # freedom.py:116
    vals = (dinv[rows] * 1.0) * dinv[cols]                                # D * A then * D (freedom.py:118)
    idx = torch.from_numpy(np.stack([rows, cols]))
    return torch.sparse_coo_tensor(idx, torch.from_numpy(vals.astype(np.float32)), (n, n), check_invariants=False)


def mgcn_norm_adj_coo(inter_row, inter_col, n_users, n_items):
    """MGCN's variant, `src/models/mgcn.py:109-144`: no epsilon, inf -> 0, everything in float32
    (the lil/dok matrices are float32, `:110`).  Returns (norm_adj N x N, R = norm_adj[:U, U:])."""
    r = np.asarray(inter_row, dtype=np.int64)
    c = np.asarray(inter_col, dtype=np.int64)
    n = n_users + n_items
    key = np.unique(np.concatenate([r * n + (c + n_users), (c + n_users) * n + r]))
    rows, cols = key // n, key % n
    rowsum = np.bincount(rows, minlength=n).astype(np.float32)            # adj.sum(1), float32
    with np.errstate(divide="ignore"):
        dinv = np.power(rowsum, np.float32(-0.5)).astype(np.float32)      # mgcn.py:121
    dinv[np.isinf(dinv)] = 0.0
    vals = ((dinv[rows] * np.float32(1.0)).astype(np.float32) * dinv[cols]).astype(np.float32)
    adj = torch.sparse_coo_tensor(torch.from_numpy(np.stack([rows, cols])), torch.from_numpy(vals), (n, n),
                                  check_invariants=False)
    m = rows < n_users                                                    # norm_adj[:U, U:] (mgcn.py:134)
    R = torch.sparse_coo_tensor(torch.from_numpy(np.stack([rows[m], cols[m] - n_users])), torch.from_numpy(vals[m]),
                                (n_users, n_items), check_invariants=False)
    return adj, R


# --------------------------------------------------------------------------------------
# a2: degree-sensitive edge pruning
# --------------------------------------------------------------------------------------


def normalize_adj_m(indices: torch.Tensor, n_users: int, n_items: int) -> torch.Tensor:
    """Per-edge 1/sqrt(d_u d_i) in fp32, `src/models/freedom.py:145-154` (same: `layergcn.py:72-81`).
    `ones_like(indices[0])` is int64, so the degree sums are exact and `1e-7 + deg` happens in fp32."""
    adj = torch.sparse_coo_tensor(indices, torch.ones_like(indices[0]), (n_users, n_items), check_invariants=False)
    row_sum = 1e-7 + torch.sparse.sum(adj, -1).to_dense()
    col_sum = 1e-7 + torch.sparse.sum(adj.t(), -1).to_dense()
    r_inv_sqrt = torch.pow(row_sum, -0.5)
    c_inv_sqrt = torch.pow(col_sum, -0.5)
    return r_inv_sqrt[indices[0]] * c_inv_sqrt[indices[1]]


def edge_info(inter_row, inter_col, n_users, n_items):
    """`src/models/freedom.py:156-162`: edges [2,E] int64 + their weights.  Edge ORDER: the reference takes
    `inter_matrix('coo').astype(np.float32)` (`freedom.py:42`); with this container's scipy (1.18) that
    `astype` canonicalises the COO (sorted by user then item, duplicates merged), with the pinned scipy 1.7.3
    it kept interaction order.  The golden vectors come from this container, so the oracle uses the canonical
    order; the order only permutes which index the multinomial draw refers to."""
    r = np.asarray(inter_row, dtype=np.int64)
    c = np.asarray(inter_col, dtype=np.int64)
    key = np.unique(r * n_items + c)
    edges = torch.from_numpy(np.stack([key // n_items, key % n_items]))
    return edges, normalize_adj_m(edges, n_users, n_items)


def pruned_adj_from_keep(edge_indices: torch.Tensor, keep_idx: torch.Tensor, n_users: int, n_items: int):
    """`src/models/freedom.py:135-143` after the multinomial draw: renormalise the kept edges in fp32,
    symmetrise -> un-coalesced, UNSORTED COO of size N x N."""
    keep = edge_indices[:, keep_idx].clone()
    vals = normalize_adj_m(keep, n_users, n_items)
    all_vals = torch.cat((vals, vals))
    keep[1] += n_users
    all_idx = torch.cat((keep, torch.flip(keep, [0])), 1)
    n = n_users + n_items
    return torch.sparse_coo_tensor(all_idx, all_vals, (n, n), check_invariants=False)


def prune_edges(edge_indices, edge_values, dropout, n_users, n_items):
    """`src/models/freedom.py:128-143` including the draw (global torch RNG, like the reference)."""
    keep_len = int(edge_values.size(0) * (1.0 - dropout))
    keep_idx = torch.multinomial(edge_values, keep_len)
    return pruned_adj_from_keep(edge_indices, keep_idx, n_users, n_items), keep_idx


# --------------------------------------------------------------------------------------
# item-item kNN graphs (init time; "next" row f4, restated because forward() consumes them)
# --------------------------------------------------------------------------------------


def freedom_knn_adj(feat: torch.Tensor, knn_k: int):
    """`src/models/freedom.py:79-100`: cosine kNN (self included), directed, sym-normalised with the
    (all-equal) out-degree; values = pow(k + 1e-7, -0.5)^2."""
    context_norm = feat.div(torch.norm(feat, p=2, dim=-1, keepdim=True))
    sim = torch.mm(context_norm, context_norm.transpose(1, 0))
    _, knn_ind = torch.topk(sim, knn_k, dim=-1)
    n = sim.size(0)
    idx0 = torch.arange(n).unsqueeze(1).expand(-1, knn_k)
    indices = torch.stack((torch.flatten(idx0), torch.flatten(knn_ind)), 0)
    adj = torch.sparse_coo_tensor(indices, torch.ones_like(indices[0]), (n, n), check_invariants=False)
    row_sum = 1e-7 + torch.sparse.sum(adj, -1).to_dense()
    r_inv_sqrt = torch.pow(row_sum, -0.5)
    values = r_inv_sqrt[indices[0]] * r_inv_sqrt[indices[1]]
    return torch.sparse_coo_tensor(indices, values, (n, n), check_invariants=False)


def freedom_mm_adj(v_feat, t_feat, knn_k, mm_image_weight):
    """`src/models/freedom.py:67-75`: w * image_adj + (1 - w) * text_adj -- a COO with DUPLICATE
    coordinates wherever both graphs share an edge (they must add)."""
    return mm_image_weight * freedom_knn_adj(v_feat, knn_k) + (1.0 - mm_image_weight) * freedom_knn_adj(t_feat, knn_k)


def mgcn_knn_adj(feat: torch.Tensor, knn_k: int):
    """`src/utils/utils.py:134-139,165-183` via `mgcn.py:56-58`: weighted (cosine) kNN graph,
    deg = scatter_add(w, row), w' = deg^-1/2[row] * w * deg^-1/2[col], inf -> 0."""
    context_norm = feat.div(torch.norm(feat, p=2, dim=-1, keepdim=True))
    sim = torch.mm(context_norm, context_norm.transpose(1, 0))
    knn_val, knn_ind = torch.topk(sim, knn_k, dim=-1)
    n = sim.shape[0]
    row = torch.arange(n).unsqueeze(1).expand(-1, knn_k).reshape(-1)
    col = knn_ind.reshape(-1)
    w = knn_val.flatten()
    deg = torch.zeros(n, dtype=w.dtype).index_add_(0, row, w)
    dis = deg.pow_(-0.5)
    dis.masked_fill_(dis == float("inf"), 0)
    w = dis[row] * w * dis[col]
    return torch.sparse_coo_tensor(torch.stack([row, col]), w, (n, n), check_invariants=False)


# --------------------------------------------------------------------------------------
# a3: propagation (forward of every graph model)
# --------------------------------------------------------------------------------------


def propagate_mean(adj, ego, n_layers):
    """E_{l+1} = A_hat E_l; mean over the L+1 layers incl. layer 0
    (`src/models/freedom.py:169-176`, `bm3.py:86-92`, `lightgcn.py:116-123`, `mgcn.py:159-166`)."""
    all_emb = [ego]
    for _ in range(n_layers):
        ego = torch.sparse.mm(adj, ego)
        all_emb += [ego]
    return torch.stack(all_emb, dim=1).mean(dim=1, keepdim=False)


def freedom_forward(adj, mm_adj, user_emb, item_emb, n_mm_layers, n_ui_layers):
    """`src/models/freedom.py:164-178`."""
    h = item_emb
    for _ in range(n_mm_layers):
        h = torch.sparse.mm(mm_adj, h)
    n_users = user_emb.shape[0]
    all_emb = propagate_mean(adj, torch.cat((user_emb, item_emb), dim=0), n_ui_layers)
    u_g, i_g = torch.split(all_emb, [n_users, item_emb.shape[0]], dim=0)
    return u_g, i_g + h


def bm3_forward(adj, user_emb, item_emb, n_layers):
    """`src/models/bm3.py:84-95` (h is the raw item id embedding, no item graph)."""
    all_emb = propagate_mean(adj, torch.cat((user_emb, item_emb), dim=0), n_layers)
    u_g, i_g = torch.split(all_emb, [user_emb.shape[0], item_emb.shape[0]], dim=0)
    return u_g, i_g + item_emb


def lightgcn_forward(adj, user_emb, item_emb, n_layers):
    """`src/models/lightgcn.py:115-128`."""
    all_emb = propagate_mean(adj, torch.cat([user_emb, item_emb], 0), n_layers)
    return all_emb[:user_emb.shape[0], :], all_emb[user_emb.shape[0]:, :]


def layergcn_forward(adj, user_emb, item_emb, n_layers):
    """`src/models/layergcn.py:125-138`: E_{l+1} = cos(A E_l, E_0) * (A E_l); SUM of layers 1..L."""
    ego = torch.cat([user_emb, item_emb], 0)
    all_emb = ego
    layers = []
    for _ in range(n_layers):
        all_emb = torch.sparse.mm(adj, all_emb)
        w = F.cosine_similarity(all_emb, ego, dim=-1)
        all_emb = torch.einsum("a,ab->ab", w, all_emb)
        layers.append(all_emb)
    out = torch.sum(torch.stack(layers, dim=0), dim=0)
    return torch.split(out, [user_emb.shape[0], item_emb.shape[0]])


def mgcn_forward(p, adj, R, image_adj, text_adj, n_ui_layers, n_layers, train=False):
    """`src/models/mgcn.py:146-207`.  `p` maps the reference's parameter names to tensors."""
    lin = lambda x, name: F.linear(x, p[name + ".weight"], p.get(name + ".bias"))
    image_feats = lin(p["image_embedding.weight"], "image_trs")
    text_feats = lin(p["text_embedding.weight"], "text_trs")
    item_w, user_w = p["item_id_embedding.weight"], p["user_embedding.weight"]
    n_users, n_items = user_w.shape[0], item_w.shape[0]
    image_item = item_w * torch.sigmoid(lin(image_feats, "gate_v.0"))           # :153
    text_item = item_w * torch.sigmoid(lin(text_feats, "gate_t.0"))             # :154
    content = propagate_mean(adj, torch.cat([user_w, item_w], dim=0), n_ui_layers)  # :157-167
    for _ in range(n_layers):
        image_item = torch.sparse.mm(image_adj, image_item)                     # :172
    image_user = torch.sparse.mm(R, image_item)                                 # :176
    image_embeds = torch.cat([image_user, image_item], dim=0)
    for _ in range(n_layers):
        text_item = torch.sparse.mm(text_adj, text_item)                        # :180
    text_user = torch.sparse.mm(R, text_item)                                   # :184
    text_embeds = torch.cat([text_user, text_item], dim=0)
    q = lambda x: F.linear(torch.tanh(lin(x, "query_common.0")), p["query_common.2.weight"])
    att = torch.cat([q(image_embeds), q(text_embeds)], dim=-1)                  # :188
    w = torch.softmax(att, dim=-1)
    common = w[:, 0].unsqueeze(1) * image_embeds + w[:, 1].unsqueeze(1) * text_embeds
    sep_i, sep_t = image_embeds - common, text_embeds - common
    sep_i = torch.sigmoid(lin(content, "gate_image_prefer.0")) * sep_i          # :195-198
    sep_t = torch.sigmoid(lin(content, "gate_text_prefer.0")) * sep_t
    side = (sep_i + sep_t + common) / 3                                         # :199
    all_embeds = content + side
    u, i = torch.split(all_embeds, [n_users, n_items], dim=0)
    if train:
        return u, i, side, content
    return u, i


def mmgcn_mean_aggregate(edge_index: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """PARITY OF THIS PRIMITIVE UNPINNED (torch_geometric is absent here): it restates PyG's documented behaviour, and so
    does the shim under which the reference's MMGCN is run for the golden file (tests/golden/ref_loader.py) -- everything
    around it (towers, loss, scoring) IS pinned to the reference's own code through tests/golden/mmgcn_tiny.npz.
    Restates `src/models/mmgcn.py:191-213` + `:40-42`: PyG `MessagePassing(aggr='mean')` with
    `message = x_j` over edge_index = [src; dst] holding both directions: out[dst] = mean_j x[src_j]."""
    src, dst = edge_index[0], edge_index[1]
    out = torch.zeros_like(x).index_add_(0, dst, x[src])
    cnt = torch.zeros(x.shape[0], dtype=x.dtype).index_add_(0, dst, torch.ones_like(dst, dtype=x.dtype))
    return out / cnt.clamp(min=1).unsqueeze(1)


def mmgcn_gcn_forward(p, prefix, edge_index, features, id_embedding, preference, dim_latent, concate=True, has_id=True):
    """One modality tower, `src/models/mmgcn.py:163-188` (`concate = 'False'` is truthy, `:31`); pinned to the reference's
    model code run under the PyG shim (tests/test_oracle_golden.py::test_mmgcn_matches_reference_model_code):
    `p` maps parameter names (`<prefix>.MLP.weight`, `<prefix>.conv_embed_1.weight`, ...) to tensors."""
    g = lambda name: p[prefix + "." + name]
    lin = lambda x, name: F.linear(x, g(name + ".weight"), g(name + ".bias"))
    temp = lin(features, "MLP") if dim_latent else features
    x = F.normalize(torch.cat((preference, temp), dim=0))
    for li in (1, 2, 3):
        h = F.leaky_relu(mmgcn_mean_aggregate(edge_index, torch.matmul(x, g(f"conv_embed_{li}.weight"))))
        x_hat = F.leaky_relu(lin(x, f"linear_layer{li}")) + id_embedding if has_id else F.leaky_relu(lin(x, f"linear_layer{li}"))
        x = F.leaky_relu(lin(torch.cat((h, x_hat), dim=1), f"g_layer{li}")) if concate else F.leaky_relu(lin(h, f"g_layer{li}") + x_hat)
    return x


def mmgcn_forward(p, edge_index, v_feat, t_feat, id_embedding, v_preference, t_preference, v_dim_latent=256):
    """`src/models/mmgcn.py:64-77`: mean of the two modality towers (the visual one with a 256-wide latent MLP, `:46-47`)."""
    rep = mmgcn_gcn_forward(p, "v_gcn", edge_index, v_feat, id_embedding, v_preference, v_dim_latent)
    rep = rep + mmgcn_gcn_forward(p, "t_gcn", edge_index, t_feat, id_embedding, t_preference, None)
    return rep / 2


def mmgcn_loss(rep, id_embedding, v_preference, batch, n_users, reg_weight):
    """`src/models/mmgcn.py:79-96`: log-sigmoid of (pos - neg) through the [1, -1] weight, plus the embedding regulariser."""
    users, pos, neg = batch[0], batch[1] + n_users, batch[2] + n_users
    user_tensor = users.repeat_interleave(2)
    item_tensor = torch.stack((pos, neg)).t().contiguous().view(-1)
    score = torch.sum(rep[user_tensor] * rep[item_tensor], dim=1).view(-1, 2)
    loss = -torch.mean(torch.log(torch.sigmoid(torch.matmul(score, torch.tensor([[1.0], [-1.0]])))))
    reg = (id_embedding[user_tensor] ** 2 + id_embedding[item_tensor] ** 2).mean() + (v_preference ** 2).mean()
    return loss + reg_weight * reg


# --------------------------------------------------------------------------------------
# a5: modality projection
# --------------------------------------------------------------------------------------


def project(table, weight, bias, idx=None, l2_normalize=False):
    """`nn.Linear` over the WHOLE feature table, gather afterwards (`src/models/freedom.py:205-209`,
    `bm3.py:102-104`, `mgcn.py:148-150`); `F.normalize` variant per `mmgcn.py:165-168`."""
    y = F.linear(table, weight, bias)
    if l2_normalize:
        y = F.normalize(y)
    return y if idx is None else y[idx]


# --------------------------------------------------------------------------------------
# losses (so that a4, the backward of the path, has an oracle through autograd)
# --------------------------------------------------------------------------------------


def bpr_loss(users, pos_items, neg_items):
    """`src/models/freedom.py:180-187`."""
    pos = torch.sum(torch.mul(users, pos_items), dim=1)
    neg = torch.sum(torch.mul(users, neg_items), dim=1)
    return -torch.mean(F.logsigmoid(pos - neg))


def freedom_loss(p, masked_adj, mm_adj, batch, n_mm_layers, n_ui_layers, reg_weight):
    """`src/models/freedom.py:189-210`."""
    users, pos, neg = batch[0], batch[1], batch[2]
    ua, ia = freedom_forward(masked_adj, mm_adj, p["user_embedding.weight"], p["item_id_embedding.weight"],
                             n_mm_layers, n_ui_layers)
    loss = bpr_loss(ua[users], ia[pos], ia[neg])
    tf = F.linear(p["text_embedding.weight"], p["text_trs.weight"], p["text_trs.bias"])
    mf_t = bpr_loss(ua[users], tf[pos], tf[neg])
    vf = F.linear(p["image_embedding.weight"], p["image_trs.weight"], p["image_trs.bias"])
    mf_v = bpr_loss(ua[users], vf[pos], vf[neg])
    return loss + reg_weight * (mf_t + mf_v)


def emb_loss(*embeddings):
    """`src/common/loss.py:38-51`."""
    out = torch.zeros(1)
    for e in embeddings:
        out = out + torch.norm(e, p=2)
    return out / embeddings[-1].shape[0]


def lightgcn_loss(p, adj, batch, n_layers, reg_weight):
    """`src/models/lightgcn.py:130-154` with `common/loss.py:9-35` (BPRLoss, gamma 1e-10)."""
    user, pos, neg = batch[0], batch[1], batch[2]
    ue, ie = p["embedding_dict.user_emb"], p["embedding_dict.item_emb"]
    ua, ia = lightgcn_forward(adj, ue, ie, n_layers)
    pos_s = torch.mul(ua[user], ia[pos]).sum(dim=1)
    neg_s = torch.mul(ua[user], ia[neg]).sum(dim=1)
    mf = -torch.log(1e-10 + torch.sigmoid(pos_s - neg_s)).mean()
    return mf + reg_weight * emb_loss(ue[user], ie[pos], ie[neg])


def layergcn_loss(p, adj, batch, n_layers, reg_weight):
    """`src/models/layergcn.py:140-174` with `common/loss.py:54-62` (L2Loss)."""
    user, pos, neg = batch[0], batch[1], batch[2]
    ue, ie = p["user_embeddings"], p["item_embeddings"]
    ua, ia = layergcn_forward(adj, ue, ie, n_layers)
    pos_s = torch.mul(ua[user], ia[pos]).sum(dim=1)
    neg_s = torch.mul(ua[user], ia[neg]).sum(dim=1)
    mf = torch.sum(-F.logsigmoid(pos_s - neg_s))
    reg = torch.zeros(1)
    for e in (ue[user], ie[pos], ie[neg]):
        reg = reg + torch.sum(e ** 2) * 0.5
    return mf + reg_weight * reg


def info_nce(view1, view2, temperature):
    """`src/models/mgcn.py:224-231`."""
    view1, view2 = F.normalize(view1, dim=1), F.normalize(view2, dim=1)
    pos = torch.exp((view1 * view2).sum(dim=-1) / temperature)
    ttl = torch.exp(torch.matmul(view1, view2.transpose(0, 1)) / temperature).sum(dim=1)
    return torch.mean(-torch.log(pos / ttl))


def mgcn_loss(p, adj, R, image_adj, text_adj, batch, n_ui_layers, n_layers, reg_weight, cl_loss, batch_size):
    """`src/models/mgcn.py:209-253`."""
    users, pos, neg = batch[0], batch[1], batch[2]
    ua, ia, side, content = mgcn_forward(p, adj, R, image_adj, text_adj, n_ui_layers, n_layers, train=True)
    u, pi, ni = ua[users], ia[pos], ia[neg]
    mf = bpr_loss(u, pi, ni)
    reg = (0.5 * (u ** 2).sum() + 0.5 * (pi ** 2).sum() + 0.5 * (ni ** 2).sum()) / batch_size
    n_users, n_items = ua.shape[0], ia.shape[0]
    side_u, side_i = torch.split(side, [n_users, n_items], dim=0)
    cont_u, cont_i = torch.split(content, [n_users, n_items], dim=0)
    cl = info_nce(side_i[pos], cont_i[pos], 0.2) + info_nce(side_u[users], cont_u[users], 0.2)
    return mf + reg_weight * reg + 0.0 + cl_loss * cl


def bm3_loss(p, adj, batch, n_layers, reg_weight, cl_weight, dropout):
    """`src/models/bm3.py:97-147`.  `F.dropout` is functional (always active) and draws from the global
    torch RNG in this order: u_target, i_target, t_feat_target, v_feat_target."""
    lin = lambda x, name: F.linear(x, p[name + ".weight"], p[name + ".bias"])
    cos = F.cosine_similarity
    u_ori, i_ori = bm3_forward(adj, p["user_embedding.weight"], p["item_id_embedding.weight"], n_layers)
    t_on = lin(p["text_embedding.weight"], "text_trs")
    v_on = lin(p["image_embedding.weight"], "image_trs")
    with torch.no_grad():
        u_t, i_t = F.dropout(u_ori.clone(), dropout), F.dropout(i_ori.clone(), dropout)
        t_t = F.dropout(t_on.clone(), dropout)
        v_t = F.dropout(v_on.clone(), dropout)
    u_on, i_on = lin(u_ori, "predictor"), lin(i_ori, "predictor")
    users, items = batch[0], batch[1]
    u_on, i_on, u_t, i_t = u_on[users, :], i_on[items, :], u_t[users, :], i_t[items, :]
    t_on = lin(t_on, "predictor")[items, :]
    t_t = t_t[items, :]
    loss_t = 1 - cos(t_on, i_t.detach(), dim=-1).mean()
    loss_tv = 1 - cos(t_on, t_t.detach(), dim=-1).mean()
    v_on = lin(v_on, "predictor")[items, :]
    v_t = v_t[items, :]
    loss_v = 1 - cos(v_on, i_t.detach(), dim=-1).mean()
    loss_vt = 1 - cos(v_on, v_t.detach(), dim=-1).mean()
    loss_ui = 1 - cos(u_on, i_t.detach(), dim=-1).mean()
    loss_iu = 1 - cos(i_on, u_t.detach(), dim=-1).mean()
    return (loss_ui + loss_iu).mean() + reg_weight * emb_loss(u_ori, i_ori) + \
        cl_weight * (loss_t + loss_v + loss_tv + loss_vt).mean()


# --------------------------------------------------------------------------------------
# a6 / a7: full-catalog scoring, mask, top-k
# --------------------------------------------------------------------------------------


def full_sort_scores(user_e, item_e, users):
    """`src/models/freedom.py:216-220` (same in bm3/mgcn/layergcn/lightgcn): S = U_g[users] I_g^T."""
    return torch.matmul(user_e[users], item_e.transpose(0, 1))


def mask_topk(scores, mask, k):
    """`src/common/trainer.py:304-309`: in-place -1e10 on the train positives, then torch.topk
    (values descending; the order among exactly equal scores is unspecified by torch)."""
    scores[mask[0], mask[1]] = -1e10
    return torch.topk(scores, k, dim=-1)


def topk_tie_low_index(scores: np.ndarray, k: int):
    """Deterministic contract of the CUDA top-k: descending score, ties broken towards the LOWER item
    index (a valid `torch.topk` answer; used to check the kernel bit-exactly on identical scores)."""
    order = np.lexsort((np.arange(scores.shape[1])[None, :].repeat(scores.shape[0], 0), -scores.astype(np.float64)), axis=1)
    idx = order[:, :k]
    return np.take_along_axis(scores, idx, 1), idx


# --------------------------------------------------------------------------------------
# the fused scorer's arithmetic, bit for bit (mmrec_b200/csrc/score_cf.cu, "exact fp32 score of one (user, item)
# pair"): whichever of its kernels serves a row, the row is the top-k of these fp32 values under float_key
# --------------------------------------------------------------------------------------

MASKED_SCORE = np.float32(-1e10)                     # value of a masked item (src/common/trainer.py:307)
_CANON_NAN = np.uint32(0x7FFFFFFF)                   # the NaN every CUDA fp32 instruction returns


def _canon_nan(x: np.ndarray) -> np.ndarray:
    x = np.array(x, dtype=np.float32, copy=True)
    x.view(np.uint32)[np.isnan(x)] = _CANON_NAN
    return x


def fmaf32(a, b, c) -> np.ndarray:
    """CUDA's `fmaf(a, b, c)` on fp32 arrays: a*b + c rounded once to nearest-even, subnormals kept, NaN canonical.

    a*b is exact in float64 (24 + 24 significand bits, exponents in range); s = a*b + c is rounded in float64 and
    TwoSum gives its exact error e.  Rounding s to float32 is then correct except when s sits exactly on a float32
    midpoint with e != 0 (the true value is off the midpoint by e): that case takes the neighbour on the side of e."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float32), np.asarray(b, np.float32), np.asarray(c, np.float32))
    with np.errstate(all="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        c64 = c.astype(np.float64)
        s = p + c64
        t = s - p
        e = (p - (s - t)) + (c64 - t)
        r = s.astype(np.float32)
        fin = np.isfinite(s)
        r64 = np.where(np.isinf(r) & fin, np.copysign(2.0 ** 128, s), r.astype(np.float64))   # overflow edge: 2^128
        o = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        mid = fin & (r64 != s) & ((r64 + o.astype(np.float64)) * 0.5 == s) & (e != 0)
        out = np.where(mid, np.where(e > 0, np.maximum(r, o), np.minimum(r, o)), r)
    return _canon_nan(out)


def cf_lpr(d: int) -> int:
    """Blocks of four elements in the chain: 8 / 16 / 32 for d <= 32 / 64 / 128."""
    return 8 if d <= 32 else (16 if d <= 64 else 32)


def cf_chain_scores(u, v) -> np.ndarray:
    """fp32 scores of u [..., d] with v [..., d] (broadcast over the leading axes) in the fused scorer's arithmetic:
    L = cf_lpr(d) blocks of four elements (zero beyond d), p_l = fmaf(u3,v3, fmaf(u2,v2, fmaf(u1,v1, fmaf(u0,v0, +0)))),
    then p_a = p_a + p_(a+w) for a < w, w = L/2 .. 1; the score is p_0."""
    u, v = np.asarray(u, np.float32), np.asarray(v, np.float32)
    d = u.shape[-1]
    assert v.shape[-1] == d and 1 <= d <= 128
    L = cf_lpr(d)
    shape = np.broadcast_shapes(u.shape[:-1], v.shape[:-1])
    zero = np.zeros(shape, np.float32)
    p = []
    for blk in range(L):
        acc = zero
        for j in range(4 * blk, 4 * blk + 4):
            # an element beyond d is fmaf(0, 0, acc) = acc + (+0): only a -0 changes (to +0)
            acc = fmaf32(u[..., j], v[..., j], acc) if j < d else (acc + np.float32(0)).astype(np.float32)
        p.append(acc)
    w = L // 2
    while w >= 1:
        for a_ in range(w):
            with np.errstate(all="ignore"):
                p[a_] = (p[a_] + p[a_ + w]).astype(np.float32)
        w //= 2
    return _canon_nan(p[0])


def float_key(x) -> np.ndarray:
    """The kernels' order-preserving uint32 key (common.cuh): ascending key = ascending value, +0 > -0, +NaN largest."""
    b = np.asarray(x, np.float32).view(np.uint32)
    return np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def topk_float_key(vals, k: int, idx=None):
    """Top-k of each row of `vals` [B, N] by float_key descending, then item index ascending (`idx` [B, N] or [N]:
    the items' indices, default 0..N-1).  Returns (values fp32 [B, k], indices int64 [B, k])."""
    vals = np.asarray(vals, np.float32)
    if idx is None:
        idx = np.arange(vals.shape[-1])
    idx = np.broadcast_to(np.asarray(idx, np.int64), vals.shape)
    order = np.lexsort((idx, np.uint32(0xFFFFFFFF) - float_key(vals)), axis=-1)[..., :k]
    return np.take_along_axis(vals, order, -1), np.take_along_axis(idx, order, -1)


def cf_exact_topk(user_e, item_e, users, mask, k: int, item_offset: int = 0, device=None, chunk_elems: int = 1 << 28):
    """What `mmrec_score_topk` (fused path) must return, bit for bit: per row the top-k of the fp32 chain scores
    (cf_chain_scores) with masked items at -1e10, by float_key then lower item index.  `mask` = [2, nnz] (batch row,
    GLOBAL item column); entries outside [0, B) x [item_offset, item_offset + n_items) are ignored, duplicates allowed.

    Emulating the chain over B x n_items is too slow on the host, so the fp64 scores s (torch, on `device`, in row chunks)
    select the candidates first.  Per pair |chain - s| <= gamma = 16 * 2^-24 * |u| * max_i |v_i| (at most 9 roundings
    on any path of the chain, Cauchy-Schwarz) + 192 * 2^-149 (underflow).  Hence the k-th largest chain value is
    >= s_(k) - gamma and every member of the fp32 top-k has s >= s_(k) - 2 gamma: only those items are emulated.
    Rows or catalogues holding a non-finite element are emulated over every item."""
    dev = torch.device("cpu") if device is None else torch.device(device)
    ue = torch.as_tensor(user_e).detach().to(dev, torch.float32)
    ie = torch.as_tensor(item_e).detach().to(dev, torch.float32)
    if users is not None:
        ue = ue[torch.as_tensor(users).to(dev, torch.int64)]
    B, d = ue.shape
    n_items = ie.shape[0]
    assert n_items >= k
    u_np, i_np = ue.cpu().numpy(), ie.cpu().numpy()
    # mask -> sorted unique (row, local item) pairs inside the batch and the shard
    if mask is not None and torch.as_tensor(mask).numel() > 0:
        m = torch.as_tensor(mask).cpu().to(torch.int64)
        mr, mc = m[0], m[1] - item_offset
        ok = (mr >= 0) & (mr < B) & (mc >= 0) & (mc < n_items)
        key = torch.unique(mr[ok] * n_items + mc[ok])
        mrow, mcol = (key // n_items).to(dev), (key % n_items).to(dev)
    else:
        mrow = mcol = torch.zeros(0, dtype=torch.int64, device=dev)
    ie64 = ie.double()
    vmax = ie64.norm(dim=1).max()
    cat_finite = bool(torch.isfinite(ie).all())
    row_finite = torch.isfinite(ue).all(dim=1).cpu().numpy()
    out_v = np.empty((B, k), np.float32)
    out_i = np.empty((B, k), np.int64)
    full_rows = np.nonzero(~row_finite)[0].tolist() if cat_finite else list(range(B))
    masked_val = float(MASKED_SCORE)
    rows_per = max(1, chunk_elems // n_items)
    pr, pi, extra = [], [], {}
    for r0 in range(0, B if cat_finite else 0, rows_per):
        r1 = min(B, r0 + rows_per)
        u64 = ue[r0:r1].double()
        s = u64 @ ie64.T
        sel = (mrow >= r0) & (mrow < r1)
        msk = torch.zeros_like(s, dtype=torch.bool)
        msk[mrow[sel] - r0, mcol[sel]] = True
        s = torch.where(msk, torch.full_like(s, masked_val), s)
        gamma = 16 * 2.0 ** -24 * u64.norm(dim=1) * vmax + 192 * 2.0 ** -149
        thr = torch.topk(s, k, dim=1).values[:, -1] - 2 * gamma
        cand = (s >= thr[:, None]) & ~msk
        rr, ii = torch.nonzero(cand, as_tuple=True)
        pr.append(rr.cpu().numpy() + r0); pi.append(ii.cpu().numpy())
        # masked items enter only when -1e10 itself is within reach; all equal, so the k lowest indices suffice
        for r in torch.nonzero(thr <= masked_val).flatten().tolist():
            extra[r0 + r] = torch.nonzero(msk[r]).flatten()[:k].cpu().numpy()
    if cat_finite:
        pr, pi = np.concatenate(pr), np.concatenate(pi)
        keep = row_finite[pr]
        pr, pi = pr[keep], pi[keep]
        vals = cf_chain_scores(u_np[pr], i_np[pi])
        starts = np.searchsorted(pr, np.arange(B + 1))          # nonzero() is row-major: pairs grouped by row
        for r in np.nonzero(row_finite)[0]:
            v, ix = vals[starts[r]:starts[r + 1]], pi[starts[r]:starts[r + 1]]
            if r in extra:
                v = np.concatenate([v, np.full(len(extra[r]), MASKED_SCORE)]); ix = np.concatenate([ix, extra[r]])
            tv, ti = topk_float_key(v[None], k, ix[None])
            out_v[r], out_i[r] = tv[0], ti[0]
    mrow_np, mcol_np = mrow.cpu().numpy(), mcol.cpu().numpy()
    for r in full_rows:                                         # every item: non-finite row or catalogue
        v = cf_chain_scores(u_np[r][None, :], i_np)
        v[mcol_np[mrow_np == r]] = MASKED_SCORE
        tv, ti = topk_float_key(v[None], k)
        out_v[r], out_i[r] = tv[0], ti[0]
    return torch.from_numpy(out_v), torch.from_numpy(out_i + item_offset)


# --------------------------------------------------------------------------------------
# evaluator ("next" row f2; needed for Recall@20 parity) -- `src/utils/topk_evaluator.py:58-102`,
# `src/utils/metrics.py:12-105`
# --------------------------------------------------------------------------------------


def topk_metrics(topk_index: np.ndarray, pos_items, topk=(5, 10, 20, 50), metrics=("recall", "ndcg", "precision", "map")):
    pos_len = np.array([len(x) for x in pos_items])
    hit = np.array([[i in set(m.tolist()) for i in n] for m, n in zip(pos_items, topk_index)])  # topk_evaluator.py:90-93
    K = hit.shape[1]
    out = {}
    res = {}
    res["recall"] = (np.cumsum(hit, axis=1) / pos_len.reshape(-1, 1)).mean(axis=0)             # metrics.py:12-15
    res["precision"] = (hit.cumsum(axis=1) / np.arange(1, K + 1)).mean(axis=0)                # metrics.py:92-105
    len_rank = np.full_like(pos_len, K)
    idcg_len = np.where(pos_len > len_rank, len_rank, pos_len)                                # metrics.py:48-66
    iranks = np.zeros_like(hit, dtype=float)
    iranks[:, :] = np.arange(1, K + 1)
    idcg = np.cumsum(1.0 / np.log2(iranks + 1), axis=1)
    for row, idx in enumerate(idcg_len):
        idcg[row, idx:] = idcg[row, idx - 1]
    dcg = np.cumsum(np.where(hit, 1.0 / np.log2(iranks + 1), 0), axis=1)
    res["ndcg"] = (dcg / idcg).mean(axis=0)
    pre = hit.cumsum(axis=1) / np.arange(1, K + 1)                                            # metrics.py:69-89
    sum_pre = np.cumsum(pre * hit.astype(float), axis=1)
    result = np.zeros_like(hit, dtype=float)
    for row, lens in enumerate(idcg_len):
        ranges = np.arange(1, K + 1)
        ranges[lens:] = ranges[lens - 1]
        result[row] = sum_pre[row] / ranges
    res["map"] = result.mean(axis=0)
    for m in metrics:
        for k in topk:
            out[f"{m}@{k}"] = round(float(res[m][k - 1]), 4)                                  # topk_evaluator.py:99-101
    return out


# --------------------------------------------------------------------------------------
# exactly representable operands: inputs on which every correct kernel returns the exact result bit for bit
# (tests/test_gpu_exact_arith.py).  Operands are integers times a power of two.  If every product is exact in fp32 and,
# for each output, sum |a||b| < 2^22 in units of the product granularity, then every partial sum of every summation
# order is an integer below 2^22 units, so an fp32 adder that keeps 24 bits after alignment never rounds: K splits,
# chunk rotations, lane widths and tilings cannot change a bit.  Epilogues that round (a division, sqrt, a product)
# are emulated below in numpy float32, whose +, -, *, / and sqrt are IEEE, correctly rounded.
# --------------------------------------------------------------------------------------

EXACT_BUDGET = 1 << 22                               # max sum |a||b| per output, in units of the product granularity


def exact_ints(rng, shape, bits, density=1.0, signed=True, full=False):
    """int64 array of `shape`: nonzero entries with at most `bits` significant bits (|m| < 2^bits), zeros elsewhere
    with probability 1 - density.  `full`: every nonzero has EXACTLY `bits` significant bits (odd, >= 2^(bits-1)),
    so a tf32 split of it into an 11-bit hi leaves a nonzero lo whenever bits > 11."""
    if full and bits == 1:
        m = np.ones(shape, dtype=np.int64)
    elif full:
        m = rng.integers(1 << (bits - 2), 1 << (bits - 1), size=shape, dtype=np.int64) * 2 + 1   # odd, in (2^(bits-1), 2^bits)
    else:
        m = rng.integers(0, 1 << bits, size=shape, dtype=np.int64)
    if signed:
        m = m * rng.choice(np.array([-1, 1], dtype=np.int64), size=shape)
    if density < 1.0:
        m = m * (rng.random(shape) < density)
    return m


def significant_bits(m) -> np.ndarray:
    """Number of bits from the highest to the lowest set bit of |m| (0 for 0)."""
    a = np.abs(np.asarray(m, dtype=np.int64))
    out = np.zeros(a.shape, dtype=np.int64)
    nz = a != 0
    if nz.any():
        v = a[nz]
        low = (v & -v)
        out[nz] = np.floor(np.log2(v.astype(np.float64))).astype(np.int64) - np.log2(low.astype(np.float64)).astype(np.int64) + 1
    return out


def to_f32_exact(m, scale: float) -> np.ndarray:
    """m * scale as float32, asserting the conversion is exact (|m| < 2^24, scale a power of two)."""
    m = np.asarray(m, dtype=np.int64)
    assert np.frexp(scale)[0] == 0.5, "scale must be a power of two"
    assert int(np.abs(m).max(initial=0)) < (1 << 24), "integer does not fit a float32 significand"
    out = (m.astype(np.float64) * scale).astype(np.float32)
    assert np.array_equal(out.astype(np.float64), m.astype(np.float64) * scale)
    return out


def int_matmul(a, b) -> np.ndarray:
    """Exact a @ b of integer matrices through float64 BLAS (numpy's int64 matmul has no BLAS): exact while every
    sum_k |a||b| is below 2^53, which is asserted."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert float((np.abs(a) @ np.abs(b)).max(initial=0.0)) < 2.0 ** 53
    return (a @ b).astype(np.int64)


def exact_matmul_bound(a, b) -> int:
    """max over outputs of sum_k |a[i,k]| |b[k,j]| for integer a [n, K] and b [K, m] (the precondition of exactness),
    after asserting every single product is exact in fp32 (< 2^24)."""
    a, b = np.abs(np.asarray(a, dtype=np.int64)), np.abs(np.asarray(b, dtype=np.int64))
    assert int(a.max(initial=0)) * int(b.max(initial=0)) < (1 << 24), "a product is not exact in fp32"
    return int(int_matmul(a, b).max(initial=0))


def assert_exact_matmul(a, b, budget: int = EXACT_BUDGET) -> None:
    s = exact_matmul_bound(a, b)
    assert s < budget, f"exactness precondition broken: sum |a||b| = {s} >= {budget} units"


def tf32_split_trunc(x):
    """K2's split of the streamed table (`split_tf32_trunc`): hi = x with the low 13 mantissa bits cleared, lo = x - hi.
    Returns (hi, lo, lo_tc): lo_tc is lo as the tensor core reads it (low 13 mantissa bits truncated)."""
    x = np.asarray(x, dtype=np.float32)
    hi = (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    lo = (x - hi).astype(np.float32)
    lo_tc = (lo.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    return hi, lo, lo_tc


def _tf32_rna(x):
    """cvt.rna.tf32.f32: round to 10 mantissa bits, ties away from zero (finite inputs)."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + np.uint64(0x1000)) & np.uint64(0xFFFFE000)).astype(np.uint32)
    return r.view(np.float32)


def tf32_split_rn(x):
    """`split_tf32` (weights of K2, both operands of K3t): hi = rna_tf32(x), lo = rna_tf32(x - hi)."""
    x = np.asarray(x, dtype=np.float32)
    hi = _tf32_rna(x)
    lo = _tf32_rna((x - hi).astype(np.float32))
    return hi, lo


def fdiv_f32(a, b) -> np.ndarray:
    """`__fdiv_rn` / IEEE `/` in fp32."""
    return (np.asarray(a, np.float32) / np.asarray(b, np.float32)).astype(np.float32)


def spmm_epilogue_f32(y, acc_in=None, acc_div: float = 1.0, post=None, gate_ref=None, y_old=None):
    """The fused SpMM epilogue of csrc/spmm.cu on an exact product y [n, d] (float32): optional LayerGCN gate
    `y *= dot / (max(sqrt(ny), 1e-8) max(sqrt(nr), 1e-8))` (dot, ny, nr must be exact: the caller asserts it), then
    Y = y (+ y_old), acc = ((y + acc_in) / acc_div) + post.  Returns (Y, acc)."""
    f = np.float32
    y = np.asarray(y, np.float32)
    if gate_ref is not None:
        r = np.asarray(gate_ref, np.float32)
        dot = (y.astype(np.float64) * r).sum(1).astype(np.float32)
        ny = (y.astype(np.float64) ** 2).sum(1).astype(np.float32)
        nr = (r.astype(np.float64) ** 2).sum(1).astype(np.float32)
        den = (np.maximum(np.sqrt(ny), f(1e-8)) * np.maximum(np.sqrt(nr), f(1e-8))).astype(np.float32)
        c = (dot / den).astype(np.float32)
        y = (y * c[:, None]).astype(np.float32)
    Y = y if y_old is None else (np.asarray(y_old, np.float32) + y).astype(np.float32)
    acc = y if acc_in is None else (y + np.asarray(acc_in, np.float32)).astype(np.float32)
    if acc_div != 1.0:
        acc = fdiv_f32(acc, f(acc_div))
    if post is not None:
        acc = (acc + np.asarray(post, np.float32)).astype(np.float32)
    return Y, acc


def l2_rows_f32(y) -> np.ndarray:
    """K2's `y * (1 / max(sqrt(sum y^2), 1e-12))` per row (the sum must be exact: the caller asserts it)."""
    y = np.asarray(y, np.float32)
    ss = (y.astype(np.float64) ** 2).sum(1).astype(np.float32)
    inv = (np.float32(1.0) / np.maximum(np.sqrt(ss), np.float32(1e-12))).astype(np.float32)
    return (y * inv[:, None]).astype(np.float32)


def adam_foreach_f32(p, g, m, v, step: int, lr: float, beta1: float, beta2: float, eps: float, weight_decay: float):
    """One step of torch 2.11's `_multi_tensor_adam` (torch.optim.Adam(foreach=True) on CUDA, no amsgrad / maximize /
    capturable) element by element in fp32: the ATen foreach kernels' operation order, with their FMAs.
        grad = fma(wd, p, grad)                    _foreach_add(grads, params, alpha=wd)
        m    = fma(1 - beta1, grad - m, m)         _foreach_lerp_(exp_avgs, grads, 1 - beta1)   (weight < 0.5 branch)
        v    = v * beta2                           _foreach_mul_(exp_avg_sqs, beta2)
        v    = fma(1 - beta2, grad * grad, v)      _foreach_addcmul_(..., value=1 - beta2)      (pointwise_op_impl)
        den  = sqrt(v) / bc2_sqrt + eps            _foreach_sqrt, _foreach_div_, _foreach_add_
        p    = fma(step_size, m / den, p)          _foreach_addcdiv_(params, exp_avgs, den, step_size)
    Python-float scalars enter the kernels rounded to fp32.  Returns new (p, m, v)."""
    f = np.float32
    p, g, m, v = (np.asarray(x, np.float32) for x in (p, g, m, v))
    if weight_decay != 0:
        g = fmaf32(f(weight_decay), p, g)
    m = fmaf32(f(1 - beta1), (g - m).astype(np.float32), m)
    v = (v * f(beta2)).astype(np.float32)
    v = fmaf32(f(1 - beta2), (g * g).astype(np.float32), v)
    bc1, bc2 = 1 - beta1 ** step, 1 - beta2 ** step
    step_size, bc2_sqrt = (lr / bc1) * -1, bc2 ** 0.5
    den = ((np.sqrt(v) / f(bc2_sqrt)).astype(np.float32) + f(eps)).astype(np.float32)
    p = fmaf32(f(step_size), (m / den).astype(np.float32), p)
    return p, m, v


def assert_bits(got, want, what: str = "") -> None:
    """`got` equals `want` element for element (`torch.equal`; NaN matches NaN at the same position).  On failure the
    message names how many elements differ and the first one.  Either side may be a tensor (any device) or an array."""
    got = got.detach().cpu() if isinstance(got, torch.Tensor) else torch.from_numpy(np.asarray(got, np.float32))
    want = want.detach().cpu() if isinstance(want, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(want, dtype=np.float32))
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.is_floating_point() and want.is_floating_point():
        nan_g, nan_w = torch.isnan(got), torch.isnan(want)
        same = torch.equal(nan_g, nan_w) and torch.equal(got.masked_fill(nan_g, 0), want.masked_fill(nan_w, 0))
    else:
        same = torch.equal(got, want)
    if not same:
        bad = ((got != want) & ~(torch.isnan(got) & torch.isnan(want))) if got.is_floating_point() else (got != want)
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements differ; first at {i}: got {got[i].item()!r}, "
                             f"want {want[i].item()!r}")


# --------------------------------------------------------------------------------------
# a5b (csrc/fuse.cu), K1c (csrc/csr.cu): the kernels' stated fp32 arithmetic, operation by operation
# --------------------------------------------------------------------------------------

def fuse_chain_f32(X, W, b=None) -> np.ndarray:
    """The pre-activations of `gate_rows_kernel` / `mgcn_fuse_kernel`: acc[n, j] = b_j (+0 without a bias), then
    acc = fmaf(W[j, k], X[n, k], acc) for k = 0 .. d-1, one correctly rounded fmaf each."""
    X, W = np.asarray(X, np.float32), np.asarray(W, np.float32)
    n, d = X.shape
    assert W.shape == (d, d)
    acc = np.zeros((n, d), np.float32) if b is None else np.broadcast_to(np.asarray(b, np.float32), (n, d)).copy()
    for k in range(d):
        acc = fmaf32(W[None, :, k], X[:, k, None], acc)
    return acc


def csr_coalesce_f32(row, col, val, n_rows: int, n_cols: int, sum_duplicates: bool = True):
    """`mmrec_csr_from_coo`: a stable sort by key = row * n_cols + col, then (sum_duplicates) one entry per key whose
    value is the sequential fp32 sum of its run in input order; `val` None counts 1.0 per entry.  Returns
    (rowptr int64 [n_rows + 1], colidx int64 [nnz], vals float32 [nnz])."""
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    val = np.ones(row.shape, np.float32) if val is None else np.asarray(val, np.float32)
    key = row.astype(np.uint64) * np.uint64(n_cols) + col.astype(np.uint64)
    order = np.argsort(key, kind="stable")
    key, val = key[order], val[order]
    if sum_duplicates and key.size:
        head = np.flatnonzero(np.concatenate([[True], key[1:] != key[:-1]]))
        ends = np.append(head[1:], key.size)
        out = val[head].copy()
        for r in range(1, int((ends - head).max())):      # r-th element of every run longer than r, added in order
            live = head + r < ends
            out[live] = (out[live] + val[head[live] + r]).astype(np.float32)
        key, val = key[head], out
    rows = (key // np.uint64(n_cols)).astype(np.int64)
    rowptr = np.searchsorted(rows, np.arange(n_rows + 1), side="left").astype(np.int64)
    return rowptr, (key % np.uint64(n_cols)).astype(np.int64), val.astype(np.float32)


def bipartite_norm_f32(users, items, n_users: int, n_items: int, eps: float = 1e-7) -> np.ndarray:
    """`mmrec_bipartite_norm_f32`: per edge fl(fl(1 / fl(sqrt(fl(float(deg_u) + eps)))) * the same for the item),
    the degree converted to fp32 with round to nearest."""
    users, items = np.asarray(users, np.int64), np.asarray(items, np.int64)
    f, eps = np.float32, np.float32(eps)

    def side(deg):
        return (f(1.0) / np.sqrt((deg.astype(np.float32) + eps).astype(np.float32))).astype(np.float32)

    ru = side(np.bincount(users, minlength=n_users))[users]
    ri = side(np.bincount(items, minlength=n_items))[items]
    return (ru * ri).astype(np.float32)
