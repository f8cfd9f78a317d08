"""LATTICE (ACM MM'21) on the H100 hot path; mirrors `src/models/lattice.py` (class `LATTICE`, the constructor, config keys,
parameter names and registration order -- `GC_Linear_list` / `Bi_Linear_list` / `dropout_list` under `ngcf`, `modal_weight`
last -- so `init_seed` gives the reference's initial weights bit for bit and a reference `state_dict` loads with
`strict=True`).  Every [I, I] matrix of the reference is a CSR here: only knn_k entries per row and modality are nonzero.

Graphs:
- `norm_adj` is `graph.build_lattice_norm_adj` (`get_adj_mat`, `:100-122`: D^-1 (A + I), not symmetric), with its transpose
  for the backward.
- `image_original_adj` / `text_original_adj` (`:66-85`) are `graph.build_mgcn_knn_adj`: the cosine kNN of the feature
  table (K7 above 128 features) with its similarities as values, symmetrically normalised, fl(fl(d_i a_ij) d_j), inf -> 0.
- The learned graph (`forward(build_item_graph=True)`, `:138-157`) is built on the batch after `pre_epoch_processing` and
  in evaluation, under autograd throughout:
  1. `image_trs(image_embedding.weight)` is `ops.project` over all rows (K2; backward K5, so `FusedAdam`'s table route
     applies to the trainable feature table);
  2. `context / ||context||` is the reference's torch expression;
  3. the top knn_k of every row of `cn cn^T` is selected by `graph.knn_normalized` (score blocks + `ops.mask_topk`, ties
     to the lower index) without autograd;
  4. one pattern P holds the union of the selected pairs of both modalities and of both original graphs; the selected
     values `<cn_i, cn_j>` are `ops.sddmm(P, cn, cn)` (backward dS cn + dS^T cn, two K1 products);
  5. `w0 A_img + w1 A_txt` over P, w = softmax(modal_weight), each position fl(fl(w0 a) + fl(w1 b)) as the dense sum
     rounds it (0 where a modality has no entry);
  6. `compute_normalized_laplacian` is `ops.csr_sym_norm` on P;
  7. `item_adj = (1 - lambda) L + lambda (w0 O_img + w1 O_txt)`: P with one autograd vector of values;
  8. `h = item_adj^n_layers item_id_embedding` is `ops.spmm_values`, differentiable w.r.t. the values and h.
- Other batches use the stored graph detached (`:158-159`).  They skip `image_trs` / `text_trs`: the reference computes
  them there and drops them, so those parameters get no gradient on these batches either way.

CF part (`:165-197`): `lightgcn` is `ops.propagate_mean` over `norm_adj`; `ngcf` keeps the reference's linears,
`leaky_relu`, bi-interaction, `nn.Dropout` and `F.normalize` around `ops.spmm`; `mf` reads the tables.  The loss is the
reference's `bpr_loss`, which divides by the configured `train_batch_size` even for a short last batch.

Evaluation: `full_sort_predict` builds the learned graph like the reference (`:229-236`), but once per evaluation through
the evaluation cache instead of once per batch, and leaves `self.item_adj` as the reference does; `full_sort_topk` is the
fused `ops.score_topk` of the base class.

Departures:
- The original graphs are built in memory at construction; the model neither reads nor writes `image_adj_{knn_k}.pt` /
  `text_adj_{knn_k}.pt`.  The reference loads those files whenever they exist, without checking that they belong to the
  same features or knn_k (`:64-85`), and writes them otherwise.
- An unknown `cf_model` raises `MMRecError` at construction (the reference's `forward` returns None and the loss fails
  later), as does `knn_k > n_items` (the reference's `torch.topk` fails on the first graph).
- `self.item_adj` is a `CSR` whose `vals` are the autograd values, not a dense tensor; `image_adj` / `text_adj` (the
  reference's dense learned kNN matrices) are not kept.
Supported: either modality alone, as in the reference: then the learned and original graphs are not weighted."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from .._lib import MMRecError
from ..common.abstract_recommender import GeneralRecommender

CF_MODELS = ("lightgcn", "mf", "ngcf")


class LATTICE(GeneralRecommender):
    _eval_cache_deps = ("norm_adj", "image_original_adj", "text_original_adj")

    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.embedding_dim = config["embedding_size"]
        self.feat_embed_dim = config["feat_embed_dim"]
        self.weight_size = config["weight_size"]
        self.knn_k = config["knn_k"]
        self.lambda_coeff = config["lambda_coeff"]
        self.cf_model = config["cf_model"]
        self.n_layers = config["n_layers"]
        self.reg_weight = config["reg_weight"]
        self.build_item_graph = True
        if self.cf_model not in CF_MODELS:
            raise MMRecError(f"LATTICE: cf_model {self.cf_model!r} is not one of {CF_MODELS}")
        if self.knn_k > self.n_items:
            raise MMRecError(f"LATTICE: knn_k = {self.knn_k} exceeds the {self.n_items} items")

        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.norm_adj = graph.build_lattice_norm_adj(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.item_adj = None

        self.n_ui_layers = len(self.weight_size)
        self.weight_size = [self.embedding_dim] + self.weight_size
        self.user_embedding = nn.Embedding(self.n_users, self.embedding_dim)
        self.item_id_embedding = nn.Embedding(self.n_items, self.embedding_dim)
        nn.init.xavier_uniform_(self.user_embedding.weight)
        nn.init.xavier_uniform_(self.item_id_embedding.weight)

        if config["cf_model"] == "ngcf":
            self.GC_Linear_list = nn.ModuleList()
            self.Bi_Linear_list = nn.ModuleList()
            self.dropout_list = nn.ModuleList()
            dropout_list = config["mess_dropout"]
            for i in range(self.n_ui_layers):
                self.GC_Linear_list.append(nn.Linear(self.weight_size[i], self.weight_size[i + 1]))
                self.Bi_Linear_list.append(nn.Linear(self.weight_size[i], self.weight_size[i + 1]))
                self.dropout_list.append(nn.Dropout(dropout_list[i]))

        # the original kNN graphs, built here every time (no image_adj_{k}.pt / text_adj_{k}.pt, module docstring)
        if self.v_feat is not None:
            self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=False)
            self.image_original_adj = graph.build_mgcn_knn_adj(self.v_feat, self.knn_k)
        if self.t_feat is not None:
            self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=False)
            self.text_original_adj = graph.build_mgcn_knn_adj(self.t_feat, self.knn_k)

        if self.v_feat is not None:
            self.image_trs = nn.Linear(self.v_feat.shape[1], self.feat_embed_dim)
        if self.t_feat is not None:
            self.text_trs = nn.Linear(self.t_feat.shape[1], self.feat_embed_dim)

        self.modal_weight = nn.Parameter(torch.Tensor([0.5, 0.5]))
        self.softmax = nn.Softmax(dim=0)

    def pre_epoch_processing(self):
        self.build_item_graph = True

    def _modalities(self):
        """(projection, feature table, original graph) of each modality present, image first."""
        mods = []
        if self.v_feat is not None:
            mods.append((self.image_trs, self.image_embedding, self.image_original_adj))
        if self.t_feat is not None:
            mods.append((self.text_trs, self.text_embedding, self.text_original_adj))
        return mods

    def build_learned_graph(self) -> ops.CSR:
        """`item_adj` of `forward(..., build_item_graph=True)` (`:136-157`) as a CSR over the union pattern P whose `vals`
        carry autograd back to `modal_weight`, the projections and the feature tables (module docstring, steps 1-7)."""
        n, k = self.n_items, self.knn_k
        mods = self._modalities()
        cns, keys = [], []
        own = torch.arange(n, device=self.device).repeat_interleave(k) * n
        for trs, emb, _ in mods:
            feats = ops.project(emb.weight, trs.weight, trs.bias)
            cn = feats.div(torch.norm(feats, p=2, dim=-1, keepdim=True))
            _, ind = graph.knn_normalized(cn.detach(), k)
            cns.append(cn)
            keys.append(own + ind.reshape(-1))
        for _, _, orig in mods:
            r, c, _ = orig.coo()
            keys.append(r * n + c)
        uniq, inv = torch.unique(torch.cat(keys), sorted=True, return_inverse=True)
        nnz = uniq.numel()
        rowptr = torch.zeros(n + 1, dtype=torch.int32, device=self.device)
        rowptr[1:] = torch.cumsum(torch.bincount(uniq // n, minlength=n), 0).to(torch.int32)
        P = ops.CSR(n, n, rowptr, (uniq % n).to(torch.int32), torch.zeros(nnz, dtype=torch.float32, device=self.device), nnz)
        parts = list(torch.split(inv, [key.numel() for key in keys]))
        learned, original = [], []
        for j, (cn, (_, _, orig)) in enumerate(zip(cns, mods)):
            sel = torch.zeros(nnz, dtype=torch.bool, device=self.device)
            sel[parts[j]] = True
            learned.append((sel, ops.sddmm(P, cn, cn)))
            o = torch.zeros(nnz, dtype=torch.float32, device=self.device)
            o[parts[len(mods) + j]] = orig.vals[:orig.nnz]
            original.append(o)
        if len(mods) == 2:
            weight = self.softmax(self.modal_weight)
            learned_vals = torch.where(learned[0][0], weight[0] * learned[0][1], 0.0) + \
                torch.where(learned[1][0], weight[1] * learned[1][1], 0.0)
            original_vals = weight[0] * original[0] + weight[1] * original[1]
        else:
            learned_vals = torch.where(learned[0][0], learned[0][1], 0.0)
            original_vals = original[0]
        laplacian = ops.csr_sym_norm(P, learned_vals)
        return P.with_values((1 - self.lambda_coeff) * laplacian + self.lambda_coeff * original_vals)

    def forward(self, adj, build_item_graph=False):
        if build_item_graph:
            self.item_adj = self.build_learned_graph()
        elif self.item_adj is None:
            raise MMRecError("LATTICE: no item graph yet: the first forward builds it (pre_epoch_processing sets build_item_graph)")
        else:
            self.item_adj = self.item_adj.with_values(self.item_adj.vals.detach())

        h = self.item_id_embedding.weight
        for _ in range(self.n_layers):
            h = ops.spmm_values(self.item_adj, self.item_adj.vals, h)

        if self.cf_model == "ngcf":
            ego_embeddings = torch.cat((self.user_embedding.weight, self.item_id_embedding.weight), dim=0)
            all_embeddings = [ego_embeddings]
            for i in range(self.n_ui_layers):
                side_embeddings = ops.spmm(adj, ego_embeddings)
                sum_embeddings = F.leaky_relu(self.GC_Linear_list[i](side_embeddings))
                bi_embeddings = torch.mul(ego_embeddings, side_embeddings)
                bi_embeddings = F.leaky_relu(self.Bi_Linear_list[i](bi_embeddings))
                ego_embeddings = sum_embeddings + bi_embeddings
                ego_embeddings = self.dropout_list[i](ego_embeddings)
                norm_embeddings = F.normalize(ego_embeddings, p=2, dim=1)
                all_embeddings += [norm_embeddings]
            all_embeddings = torch.stack(all_embeddings, dim=1)
            all_embeddings = all_embeddings.mean(dim=1, keepdim=False)
            u_g_embeddings, i_g_embeddings = torch.split(all_embeddings, [self.n_users, self.n_items], dim=0)
            return u_g_embeddings, i_g_embeddings + F.normalize(h, p=2, dim=1)
        if self.cf_model == "lightgcn":
            ego_embeddings = torch.cat((self.user_embedding.weight, self.item_id_embedding.weight), dim=0)
            all_embeddings = ops.propagate_mean(adj, ego_embeddings, self.n_ui_layers)
            u_g_embeddings, i_g_embeddings = torch.split(all_embeddings, [self.n_users, self.n_items], dim=0)
            return u_g_embeddings, i_g_embeddings + F.normalize(h, p=2, dim=1)
        return self.user_embedding.weight, self.item_id_embedding.weight + F.normalize(h, p=2, dim=1)

    def bpr_loss(self, users, pos_items, neg_items):
        pos_scores = torch.sum(torch.mul(users, pos_items), dim=1)
        neg_scores = torch.sum(torch.mul(users, neg_items), dim=1)
        regularizer = 1. / 2 * (users ** 2).sum() + 1. / 2 * (pos_items ** 2).sum() + 1. / 2 * (neg_items ** 2).sum()
        regularizer = regularizer / self.batch_size
        maxi = F.logsigmoid(pos_scores - neg_scores)
        mf_loss = -torch.mean(maxi)
        emb_loss = self.reg_weight * regularizer
        reg_loss = 0.0
        return mf_loss, emb_loss, reg_loss

    def calculate_loss(self, interaction):
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        ua_embeddings, ia_embeddings = self.forward(self.norm_adj, build_item_graph=self.build_item_graph)
        self.build_item_graph = False
        mf_loss, emb_loss, reg_loss = self.bpr_loss(ua_embeddings[users], ia_embeddings[pos_items], ia_embeddings[neg_items])
        return mf_loss + emb_loss + reg_loss

    def _score_embeddings(self):
        return self._cached_eval_embeddings(lambda: self.forward(self.norm_adj, build_item_graph=True))

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
