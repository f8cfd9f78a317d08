"""MMGCF (multimodal graph collaborative filtering: LightGCN with late-fused modality features) on the H100 hot path.
Same class name, constructor, config keys, parameter names, construction order and `state_dict` order as
`src/models/mmgcf.py`, so `init_seed` gives the reference's initial weights bit for bit and a reference `state_dict`
loads with `strict=True`.

Kernels:
- `norm_adj` is `graph.build_norm_adj` (`get_norm_adj_mat`, `:93-118`: `(A > 0)` degrees plus 1e-7) and
  `pre_epoch_processing` is `graph.EdgePruner.sample` (`:132-154`, FREEDOM's degree-sensitive draw and rebuild).
- Training (`calculate_loss`, `:270-284`): `ops.propagate_mean` on the masked adjacency; both modality projections as
  `ops.project` of only the 2B rows the loss reads (`both = cat(pos, neg)`; the tables are frozen, so the backward is
  K5's weight gradient alone); the fusion as `ops.late_fuse` on those rows, which gathers the propagated item rows
  itself.  Every fusion mode is row-wise, so the rows the loss reads, and the weight and bias gradients, are those of the
  reference's full-table `forward` (the rows it never reads contribute exact zeros).
- Inference (`full_sort_predict`, `:286-289`, under the evaluation cache): `ops.propagate_mean_fused` from the two
  embedding tables, K2 over both whole tables, `ops.late_fuse` over all items, `ops.score`; `full_sort_topk` inherited.
- `fusion_mode: concat` ends in an `nn.Linear` of a concatenation of at most 3 x 64 columns: it stays the reference's
  torch expression (`torch.cat` and its linears), on the gathered rows in training and on all rows in inference.

Departures from the reference (refused with `MMRecError` at construction, where the reference goes on):
- a `weighting` outside equal | alpha | normalized (the reference silently takes its `equal` branch, `:244`);
- a `fusion_mode` outside mean | sum | concat (the reference builds no concat layers and fails on the first forward in its
  `concat` branch, `:175`);
- `mean` / `sum` with `feat_embed_dim != embedding_size` (the reference fails inside `torch.stack` on the first
  forward), or with an `embedding_size` outside 32 | 64 | 128, the widths the fusion kernel has.
Either modality alone works (`n_modalities` = 1: no `mm_concat_layer`, and `equal` skips its first stage)."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from .._lib import MMRecError
from ..common.abstract_recommender import GeneralRecommender

FUSION_MODES = ("mean", "sum", "concat")
WEIGHTINGS = ("equal", "alpha", "normalized")


class MMGCF(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.embedding_dim = config["embedding_size"]
        self.feat_embed_dim = config["feat_embed_dim"]
        self.n_ui_layers = config["n_ui_layers"]
        self.reg_weight = config["reg_weight"]
        self.fusion_mode = config["fusion_mode"]
        self.weighting = config["weighting"]
        self.dropout = config["dropout"]
        if self.fusion_mode not in FUSION_MODES:
            raise MMRecError(f"MMGCF: fusion_mode {self.fusion_mode!r} is not one of {FUSION_MODES}")
        if self.weighting not in WEIGHTINGS:
            raise MMRecError(f"MMGCF: weighting {self.weighting!r} is not one of {WEIGHTINGS}")
        if self.fusion_mode != "concat":
            if self.feat_embed_dim != self.embedding_dim:
                raise MMRecError(f"MMGCF: fusion_mode {self.fusion_mode!r} needs feat_embed_dim == embedding_size, got "
                                 f"{self.feat_embed_dim} and {self.embedding_dim}")
            if self.embedding_dim not in (32, 64, 128):
                raise MMRecError(f"MMGCF: fusion_mode {self.fusion_mode!r} runs at embedding_size 32, 64 or 128, not "
                                 f"{self.embedding_dim}")

        self.n_nodes = self.n_users + self.n_items
        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.norm_adj = graph.build_norm_adj(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.masked_adj = None
        self.pruner = graph.EdgePruner(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.edge_indices, self.edge_values = self.pruner.edge_indices, self.pruner.edge_values

        self.user_embedding = nn.Embedding(self.n_users, self.embedding_dim)
        self.item_id_embedding = nn.Embedding(self.n_items, self.embedding_dim)
        nn.init.xavier_uniform_(self.user_embedding.weight)
        nn.init.xavier_uniform_(self.item_id_embedding.weight)

        self.n_modalities = 0
        if self.v_feat is not None:
            self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=True)
            self.image_trs = nn.Linear(self.v_feat.shape[1], self.feat_embed_dim)
            self.n_modalities += 1
        if self.t_feat is not None:
            self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=True)
            self.text_trs = nn.Linear(self.t_feat.shape[1], self.feat_embed_dim)
            self.n_modalities += 1

        if self.weighting == "alpha":
            self.mm_alpha = nn.Parameter(torch.tensor(0.0))

        # built for every weighting under concat, used or not: their initialisation draws from the RNG (mmgcf.py:70-85)
        if self.fusion_mode == "concat" and self.n_modalities > 0:
            all_in = self.embedding_dim + self.n_modalities * self.feat_embed_dim
            self.all_concat_layer = nn.Linear(all_in, self.embedding_dim)
            if self.n_modalities > 1:
                self.mm_concat_layer = nn.Linear(self.n_modalities * self.feat_embed_dim, self.feat_embed_dim)
            self.id_mm_concat_layer = nn.Linear(self.embedding_dim + self.feat_embed_dim, self.embedding_dim)

    def pre_epoch_processing(self):
        if self.dropout <= 0.0:
            self.masked_adj = self.norm_adj
            return
        self.masked_adj, _ = self.pruner.sample(self.dropout)

    def _mm_feats(self, idx=None):
        """The projected modality rows (`_get_mm_feats`, `:158-165`), of the items `idx` only when given: K2."""
        feats = []
        if self.v_feat is not None:
            feats.append(ops.project(self.image_embedding.weight, self.image_trs.weight, self.image_trs.bias, idx=idx))
        if self.t_feat is not None:
            feats.append(ops.project(self.text_embedding.weight, self.text_trs.weight, self.text_trs.bias, idx=idx))
        return feats

    def _concat_fusion(self, item_emb, feats):
        """`fuse_item_embeddings` (`:177-254`) under `fusion_mode: concat`, the reference's torch expression."""
        if self.weighting == "alpha":
            alpha = torch.sigmoid(self.mm_alpha)
            tensors = [item_emb * alpha] + [f * (1.0 - alpha) for f in feats]
            return self.all_concat_layer(torch.cat(tensors, dim=-1))
        if self.weighting == "normalized":
            tensors = [F.normalize(item_emb) * self.n_modalities] + [F.normalize(f) for f in feats]
            return self.all_concat_layer(torch.cat(tensors, dim=-1))
        mm_fused = self.mm_concat_layer(torch.cat(feats, dim=-1)) if len(feats) > 1 else feats[0]
        return self.id_mm_concat_layer(torch.cat([item_emb, mm_fused], dim=-1))

    def fuse_item_embeddings(self, item_emb, feats, idx=None):
        """The fused rows `item_emb[idx]` (all rows when idx is None) with `feats`, the modality rows of the same items."""
        if self.fusion_mode == "concat":
            return self._concat_fusion(item_emb if idx is None else item_emb[idx], feats)
        alpha = torch.sigmoid(self.mm_alpha).reshape(1) if self.weighting == "alpha" else None
        v = feats[0] if self.v_feat is not None else None
        t = feats[-1] if self.t_feat is not None else None
        return ops.late_fuse(item_emb, v, t, self.fusion_mode, self.weighting, alpha=alpha, idx=idx)

    def lightgcn_propagate(self, adj):
        """mean(E_0 .. E_L) of `[user_embedding; item_id_embedding]` (`:124-142`) as (user rows, item rows)."""
        user_w, item_w = self.user_embedding.weight, self.item_id_embedding.weight
        if not torch.is_grad_enabled() and user_w.is_cuda:
            # inference: layer 1 reads the two tables in place (no concatenated copy)
            out = ops.propagate_mean_fused(adj, (user_w, item_w), self.n_ui_layers, cooperative=False)
        else:
            out = ops.propagate_mean(adj, torch.cat([user_w, item_w], dim=0), self.n_ui_layers)
        return torch.split(out, [self.n_users, self.n_items], dim=0)

    def forward(self, adj):
        user_emb, item_emb = self.lightgcn_propagate(adj)
        return user_emb, self.fuse_item_embeddings(item_emb, self._mm_feats())

    def bpr_loss(self, users, pos_items, neg_items):
        pos_scores = (users * pos_items).sum(dim=1)
        neg_scores = (users * neg_items).sum(dim=1)
        return -F.logsigmoid(pos_scores - neg_scores).mean()

    def calculate_loss(self, interaction):
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        ua_emb, ia_emb = self.lightgcn_propagate(self.masked_adj)
        both = torch.cat((pos_items, neg_items))
        fused = self.fuse_item_embeddings(ia_emb, self._mm_feats(both), idx=both)   # only the rows the loss reads
        n = pos_items.numel()
        mf_loss = self.bpr_loss(ua_emb[users], fused[:n], fused[n:])
        reg_loss = (
            self.user_embedding.weight[users].norm(2).pow(2)
            + self.item_id_embedding.weight[pos_items].norm(2).pow(2)
            + self.item_id_embedding.weight[neg_items].norm(2).pow(2)
        ) / (2 * len(users))
        return mf_loss + self.reg_weight * reg_loss

    def _score_embeddings(self):
        return self._cached_eval_embeddings(lambda: self.forward(self.norm_adj))

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
