"""BM3 on the H100 hot path; mirrors `src/models/bm3.py` (class name, config keys, parameter
names and order).  forward `:84-95` -> ops.propagate_mean; projections `:102-104` -> ops.project over the whole
table (the dropout targets `:110-119` draw a mask over the whole projected table, so the gather cannot move in
front of it without changing the RNG stream); full_sort_predict `:149-154` -> predictor + ops.score."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.functional import cosine_similarity

from .. import graph, ops
from ..common.abstract_recommender import GeneralRecommender
from ..common.loss import EmbLoss


class BM3(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.embedding_dim = config["embedding_size"]
        self.feat_embed_dim = config["embedding_size"]
        self.n_layers = config["n_layers"]
        self.reg_weight = config["reg_weight"]
        self.cl_weight = config["cl_weight"]
        self.dropout = config["dropout"]
        self.n_nodes = self.n_users + self.n_items
        self.norm_adj = graph.build_norm_adj(dataset.inter_matrix(form="coo").astype(np.float32), self.n_users,
                                             self.n_items, self.device)
        self.user_embedding = nn.Embedding(self.n_users, self.embedding_dim)
        self.item_id_embedding = nn.Embedding(self.n_items, self.embedding_dim)
        nn.init.xavier_uniform_(self.user_embedding.weight)
        nn.init.xavier_uniform_(self.item_id_embedding.weight)
        self.predictor = nn.Linear(self.embedding_dim, self.embedding_dim)
        self.reg_loss = EmbLoss()
        nn.init.xavier_normal_(self.predictor.weight)
        if self.v_feat is not None:
            self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=False)
            self.image_trs = nn.Linear(self.v_feat.shape[1], self.feat_embed_dim)
            nn.init.xavier_normal_(self.image_trs.weight)
        if self.t_feat is not None:
            self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=False)
            self.text_trs = nn.Linear(self.t_feat.shape[1], self.feat_embed_dim)
            nn.init.xavier_normal_(self.text_trs.weight)

    def forward(self):
        h = self.item_id_embedding.weight
        if not torch.is_grad_enabled() and h.is_cuda:                # inference: the layers read the two tables in place
            all_emb = ops.propagate_mean_fused(self.norm_adj, (self.user_embedding.weight, h), self.n_layers, cooperative=False)
        else:
            all_emb = ops.propagate_mean(self.norm_adj, torch.cat((self.user_embedding.weight, h), dim=0), self.n_layers)
        u_g, i_g = torch.split(all_emb, [self.n_users, self.n_items], dim=0)
        return u_g, i_g + h

    def calculate_loss(self, interactions):
        """`bm3.py:97-147`.  The graph encoder and the two projections run on the hot-path kernels; what follows them
        (`_objective`) is row-wise torch arithmetic on [N, d] tensors, kept op for op in the reference's order because
        the dropout targets consume the RNG stream and the loss is compared bit for bit."""
        u_all, i_all = self.forward()
        t_proj = v_proj = None
        if self.t_feat is not None:
            t_proj = ops.project(self.text_embedding.weight, self.text_trs.weight, self.text_trs.bias)
        if self.v_feat is not None:
            v_proj = ops.project(self.image_embedding.weight, self.image_trs.weight, self.image_trs.bias)
        return self._objective(u_all, i_all, t_proj, v_proj, interactions[0], interactions[1])

    @staticmethod
    def _apart(online, target):
        """1 - mean cosine similarity of the online view to a stop-gradient target (`bm3.py:134-146`)."""
        return 1 - cosine_similarity(online, target.detach(), dim=-1).mean()

    def _objective(self, u_all, i_all, t_proj, v_proj, users, items):
        # targets: dropout views of the online embeddings, drawn in the reference's order (users, items, text, image)
        with torch.no_grad():
            u_target, i_target = u_all.clone(), i_all.clone()
            u_target = F.dropout(u_target, self.dropout)
            i_target = F.dropout(i_target, self.dropout)
            t_target = None if t_proj is None else F.dropout(t_proj.clone(), self.dropout)
            v_target = None if v_proj is None else F.dropout(v_proj.clone(), self.dropout)
        u_online, i_online = self.predictor(u_all), self.predictor(i_all)
        u_online, i_online = u_online[users, :], i_online[items, :]
        u_target, i_target = u_target[users, :], i_target[items, :]
        # per modality: (feature view vs. id target, feature view vs. its own dropout target)
        loss_t = loss_tv = loss_v = loss_vt = 0.0
        if t_proj is not None:
            t_online = self.predictor(t_proj)[items, :]
            loss_t, loss_tv = self._apart(t_online, i_target), self._apart(t_online, t_target[items, :])
        if v_proj is not None:
            v_online = self.predictor(v_proj)[items, :]
            loss_v, loss_vt = self._apart(v_online, i_target), self._apart(v_online, v_target[items, :])
        align = (self._apart(u_online, i_target) + self._apart(i_online, u_target)).mean()
        reg = self.reg_weight * self.reg_loss(u_all, i_all)
        modal = self.cl_weight * (loss_t + loss_v + loss_tv + loss_vt).mean()
        return align + reg + modal

    def _score_embeddings(self):
        def run():
            u, i = self.forward()
            return self.predictor(u), self.predictor(i)
        return self._cached_eval_embeddings(run)

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
