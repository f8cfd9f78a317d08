"""FREEDOM on the H100 hot path.  Same class name, constructor, config keys, parameter names and registration
order as `src/models/freedom.py` (so `init_seed` reproduces the same initial weights and a
reference `state_dict` loads), with the three op families delegated to `mmrec_b200.ops`:

  forward            `freedom.py:164-178`  -> ops.spmm / ops.propagate_mean (CSR SpMM, fused mean and `+ h`)
  pre_epoch_processing `freedom.py:128-143` -> graph.EdgePruner (same multinomial draw, kernels after it)
  calculate_loss     `freedom.py:189-210`  -> ops.project fused gather+linear for the modality BPR terms
  full_sort_predict  `freedom.py:212-220`  -> ops.score (fresh [B, n_items] tensor, caller may mutate it)
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from ..common.abstract_recommender import GeneralRecommender


class FREEDOM(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.embedding_dim = config["embedding_size"]
        self.feat_embed_dim = config["feat_embed_dim"]
        self.knn_k = config["knn_k"]
        self.lambda_coeff = config["lambda_coeff"]
        self.cf_model = config["cf_model"]
        self.n_layers = config["n_mm_layers"]
        self.n_ui_layers = config["n_ui_layers"]
        self.reg_weight = config["reg_weight"]
        self.build_item_graph = True
        self.mm_image_weight = config["mm_image_weight"]
        self.dropout = config["dropout"]
        self.degree_ratio = config["degree_ratio"]
        self.n_nodes = self.n_users + self.n_items

        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.norm_adj = graph.build_norm_adj(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.masked_adj, self.mm_adj = None, None
        self.pruner = graph.EdgePruner(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.edge_indices, self.edge_values = self.pruner.edge_indices, self.pruner.edge_values

        self.user_embedding = nn.Embedding(self.n_users, self.embedding_dim)
        self.item_id_embedding = nn.Embedding(self.n_items, self.embedding_dim)
        nn.init.xavier_uniform_(self.user_embedding.weight)
        nn.init.xavier_uniform_(self.item_id_embedding.weight)
        if self.v_feat is not None:
            self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=False)
            self.image_trs = nn.Linear(self.v_feat.shape[1], self.feat_embed_dim)
        if self.t_feat is not None:
            self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=False)
            self.text_trs = nn.Linear(self.t_feat.shape[1], self.feat_embed_dim)
        # item-item graph, frozen after construction (the reference caches it as a .pt next to the data)
        self.mm_adj = graph.build_freedom_mm_adj(self.v_feat, self.t_feat, self.knn_k, self.mm_image_weight)

    def pre_epoch_processing(self):
        if self.dropout <= 0.0:
            self.masked_adj = self.norm_adj
            return
        self.masked_adj, _ = self.pruner.sample(self.dropout)

    def forward(self, adj):
        ego = torch.cat((self.user_embedding.weight, self.item_id_embedding.weight), dim=0)
        if ops.CHAIN and not torch.is_grad_enabled() and self.n_layers >= 1 and self.n_ui_layers >= 1:
            # inference: the item-item product(s), the UI layers, the layer mean and `i_g + h` in one cooperative launch
            all_emb = ops.propagate_mean_fused(adj, ego, self.n_ui_layers, post_csr=self.mm_adj, post_x=self.item_id_embedding.weight,
                                               post_layers=self.n_layers, post_row0=self.n_users)
            return torch.split(all_emb, [self.n_users, self.n_items], dim=0)
        all_emb = ops.propagate_mean(adj, ego, self.n_ui_layers)
        u_g, i_g = torch.split(all_emb, [self.n_users, self.n_items], dim=0)
        if self.n_layers == 0:
            return u_g, i_g + self.item_id_embedding.weight
        h = self.item_id_embedding.weight
        for _ in range(self.n_layers - 1):
            h = ops.spmm(self.mm_adj, h)
        return u_g, ops.spmm(self.mm_adj, h, base=i_g)        # i_g + mm_adj @ h, fused

    def bpr_loss(self, users, pos_items, neg_items):
        pos = torch.sum(torch.mul(users, pos_items), dim=1)
        neg = torch.sum(torch.mul(users, neg_items), dim=1)
        return -torch.mean(F.logsigmoid(pos - neg))

    def calculate_loss(self, interaction):
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        ua, ia = self.forward(self.masked_adj)
        self.build_item_graph = False
        u = ua[users]
        loss = self.bpr_loss(u, ia[pos_items], ia[neg_items])
        mf_v, mf_t = 0.0, 0.0
        both = torch.cat((pos_items, neg_items))
        n = pos_items.numel()
        if self.t_feat is not None:
            tf = ops.project(self.text_embedding.weight, self.text_trs.weight, self.text_trs.bias, idx=both)
            mf_t = self.bpr_loss(u, tf[:n], tf[n:])
        if self.v_feat is not None:
            vf = ops.project(self.image_embedding.weight, self.image_trs.weight, self.image_trs.bias, idx=both)
            mf_v = self.bpr_loss(u, vf[:n], vf[n:])
        return loss + self.reg_weight * (mf_t + mf_v)

    def _score_embeddings(self):
        return self._cached_eval_embeddings(lambda: self.forward(self.norm_adj))

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
