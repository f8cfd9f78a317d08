"""LightGCN on the H100 hot path; mirrors `src/models/lightgcn.py` (class name, config keys,
`embedding_dict` parameter names).  forward `:115-128` -> ops.propagate_mean; full_sort_predict `:156-164` -> ops.score."""
import numpy as np
import torch
import torch.nn as nn

from .. import graph, ops
from ..common.abstract_recommender import GeneralRecommender
from ..common.loss import BPRLoss, EmbLoss


class LightGCN(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.latent_dim = config["embedding_size"]
        self.n_layers = config["n_layers"]
        self.reg_weight = config["reg_weight"]
        self.mf_loss = BPRLoss()
        self.reg_loss = EmbLoss()
        init = nn.init.xavier_uniform_
        self.embedding_dict = nn.ParameterDict({
            "user_emb": nn.Parameter(init(torch.empty(self.n_users, self.latent_dim))),
            "item_emb": nn.Parameter(init(torch.empty(self.n_items, self.latent_dim)))})
        self.norm_adj_matrix = graph.build_norm_adj(self.interaction_matrix, self.n_users, self.n_items, self.device)

    def get_ego_embeddings(self):
        return torch.cat([self.embedding_dict["user_emb"], self.embedding_dict["item_emb"]], 0)

    def forward(self):
        all_emb = ops.propagate_mean(self.norm_adj_matrix, self.get_ego_embeddings(), self.n_layers)
        return all_emb[:self.n_users, :], all_emb[self.n_users:, :]

    def calculate_loss(self, interaction):
        user, pos_item, neg_item = interaction[0], interaction[1], interaction[2]
        ua, ia = self.forward()
        u = ua[user, :]
        pos_scores = torch.mul(u, ia[pos_item, :]).sum(dim=1)
        neg_scores = torch.mul(u, ia[neg_item, :]).sum(dim=1)
        mf_loss = self.mf_loss(pos_scores, neg_scores)
        reg = self.reg_loss(self.embedding_dict["user_emb"][user, :], self.embedding_dict["item_emb"][pos_item, :],
                            self.embedding_dict["item_emb"][neg_item, :])
        return mf_loss + self.reg_weight * reg

    def _score_embeddings(self):
        return self._cached_eval_embeddings(self.forward)

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
