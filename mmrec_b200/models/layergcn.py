"""LayerGCN on the H100 hot path; mirrors `src/models/layergcn.py` (the upstream file imports a
non-existent `models.common`, `:12-13`; this one imports the real base).  forward `:125-138`: the cosine gate is
fused into the SpMM epilogue for inference; training uses SpMM + torch ops so autograd sees the gate."""
import random

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from ..common.abstract_recommender import GeneralRecommender
from ..common.loss import BPRLoss, L2Loss


class LayerGCN(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.latent_dim = config["embedding_size"]
        self.n_layers = config["n_layers"]
        self.reg_weight = config["reg_weight"]
        self.dropout = config["dropout"]
        self.n_nodes = self.n_users + self.n_items
        self.user_embeddings = nn.Parameter(nn.init.xavier_uniform_(torch.empty(self.n_users, self.latent_dim)))
        self.item_embeddings = nn.Parameter(nn.init.xavier_uniform_(torch.empty(self.n_items, self.latent_dim)))
        self.norm_adj_matrix = graph.build_norm_adj(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.masked_adj = None
        self.forward_adj = None
        self.pruning_random = False
        self.pruner = graph.EdgePruner(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.edge_indices, self.edge_values = self.pruner.edge_indices, self.pruner.edge_values
        self.mf_loss = BPRLoss()
        self.reg_loss = L2Loss()

    def pre_epoch_processing(self):
        if self.dropout <= 0.0:
            self.masked_adj = self.norm_adj_matrix
            return
        keep_len = int(self.edge_values.size(0) * (1.0 - self.dropout))
        if self.pruning_random:       # alternate uniform / degree-sensitive pruning (layergcn.py:55-61)
            keep_idx = torch.tensor(random.sample(range(self.edge_values.size(0)), keep_len), device=self.edge_values.device)
        else:
            keep_idx = torch.multinomial(self.edge_values, keep_len)
        self.pruning_random = True ^ self.pruning_random
        self.masked_adj = self.pruner.adj_from_keep(keep_idx)

    def get_ego_embeddings(self):
        return torch.cat([self.user_embeddings, self.item_embeddings], 0)

    def forward(self):
        ego = self.get_ego_embeddings()
        if not torch.is_grad_enabled():
            out = ops.propagate_layergcn(self.forward_adj, ego, self.n_layers)
        else:
            all_emb, layers = ego, []
            for _ in range(self.n_layers):
                all_emb = ops.spmm(self.forward_adj, all_emb)
                w = F.cosine_similarity(all_emb, ego, dim=-1)
                all_emb = torch.einsum("a,ab->ab", w, all_emb)
                layers.append(all_emb)
            out = torch.sum(torch.stack(layers, dim=0), dim=0)
        return torch.split(out, [self.n_users, self.n_items])

    def bpr_loss(self, u_embeddings, i_embeddings, user, pos_item, neg_item):
        u = u_embeddings[user]
        pos_scores = torch.mul(u, i_embeddings[pos_item]).sum(dim=1)
        neg_scores = torch.mul(u, i_embeddings[neg_item]).sum(dim=1)
        return torch.sum(-F.logsigmoid(pos_scores - neg_scores))

    def emb_loss(self, user, pos_item, neg_item):
        return self.reg_loss(self.user_embeddings[user], self.item_embeddings[pos_item], self.item_embeddings[neg_item])

    def calculate_loss(self, interaction):
        user, pos_item, neg_item = interaction[0], interaction[1], interaction[2]
        self.forward_adj = self.masked_adj
        ua, ia = self.forward()
        return self.bpr_loss(ua, ia, user, pos_item, neg_item) + self.reg_weight * self.emb_loss(user, pos_item, neg_item)

    def _score_embeddings(self):
        def run():
            self.forward_adj = self.norm_adj_matrix
            return self.forward()
        return self._cached_eval_embeddings(run)

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
