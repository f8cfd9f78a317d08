"""MGCN on the H100 hot path; mirrors `src/models/mgcn.py` (class name, config keys, parameter
names and order).  Six SpMMs per forward (`:157-185`) -> ops.propagate_mean / ops.spmm on CSR; projections
`:148-150` -> ops.project; the row-wise fusion (`:153-201`: purifier gates, 2-way attention, preference gates) is two
kernels at inference (`ops.gate_rows`, `ops.mgcn_fuse`, SURVEY.md 8a a5b) and torch expressions under autograd."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from ..common.abstract_recommender import GeneralRecommender


class MGCN(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.sparse = True
        self.cl_loss = config["cl_loss"]
        self.n_ui_layers = config["n_ui_layers"]
        self.embedding_dim = config["embedding_size"]
        self.knn_k = config["knn_k"]
        self.n_layers = config["n_layers"]
        self.reg_weight = config["reg_weight"]
        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.user_embedding = nn.Embedding(self.n_users, self.embedding_dim)
        self.item_id_embedding = nn.Embedding(self.n_items, self.embedding_dim)
        nn.init.xavier_uniform_(self.user_embedding.weight)
        nn.init.xavier_uniform_(self.item_id_embedding.weight)
        self.norm_adj = graph.build_norm_adj(self.interaction_matrix, self.n_users, self.n_items, self.device, variant="mgcn")
        self.R = graph.build_mgcn_R(self.interaction_matrix, self.n_users, self.n_items, self.device)
        if self.v_feat is not None:
            self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=False)
            self.image_original_adj = graph.build_mgcn_knn_adj(self.image_embedding.weight.detach(), self.knn_k)
        if self.t_feat is not None:
            self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=False)
            self.text_original_adj = graph.build_mgcn_knn_adj(self.text_embedding.weight.detach(), self.knn_k)
        if self.v_feat is not None:
            self.image_trs = nn.Linear(self.v_feat.shape[1], self.embedding_dim)
        if self.t_feat is not None:
            self.text_trs = nn.Linear(self.t_feat.shape[1], self.embedding_dim)
        self.softmax = nn.Softmax(dim=-1)
        d = self.embedding_dim
        self.query_common = nn.Sequential(nn.Linear(d, d), nn.Tanh(), nn.Linear(d, 1, bias=False))
        self.gate_v = nn.Sequential(nn.Linear(d, d), nn.Sigmoid())
        self.gate_t = nn.Sequential(nn.Linear(d, d), nn.Sigmoid())
        self.gate_image_prefer = nn.Sequential(nn.Linear(d, d), nn.Sigmoid())
        self.gate_text_prefer = nn.Sequential(nn.Linear(d, d), nn.Sigmoid())
        self.tau = 0.5

    def pre_epoch_processing(self):
        pass

    def _forward_inference(self, adj):
        """`forward` without autograd (evaluation): a5b -- the purifier gates as one kernel per modality, the modality SpMMs
        writing straight into the [users; items] tables, attention + preference gates + `content + side` as one kernel."""
        d, U = self.embedding_dim, self.n_users
        item_w = self.item_id_embedding.weight
        image_feats = ops.project(self.image_embedding.weight, self.image_trs.weight, self.image_trs.bias)
        text_feats = ops.project(self.text_embedding.weight, self.text_trs.weight, self.text_trs.bias)
        content = ops.propagate_mean(adj, torch.cat([self.user_embedding.weight, item_w], dim=0), self.n_ui_layers)
        views = []
        for feats, gate, knn in ((image_feats, self.gate_v, self.image_original_adj), (text_feats, self.gate_t, self.text_original_adj)):
            emb = torch.empty(U + self.n_items, d, dtype=torch.float32, device=item_w.device)
            x = ops.gate_rows(feats, gate[0].weight, gate[0].bias, mul=item_w, out=emb[U:] if self.n_layers == 0 else None)
            for l in range(self.n_layers):                           # mgcn.py:169-172 / :177-180
                y = emb[U:] if l == self.n_layers - 1 else torch.empty_like(x)
                ops.spmm_raw(knn, x, Y=y)
                x = y
            ops.spmm_raw(self.R, emb[U:], Y=emb[:U])                 # user rows = R @ item rows (mgcn.py:173,181)
            views.append(emb)
        q = self.query_common
        all_embeds = ops.mgcn_fuse(views[0], views[1], content, q[0].weight, q[0].bias, q[2].weight, self.gate_image_prefer[0].weight,
                                   self.gate_image_prefer[0].bias, self.gate_text_prefer[0].weight, self.gate_text_prefer[0].bias)
        return all_embeds[:U], all_embeds[U:]

    def forward(self, adj, train=False):
        if not train and not torch.is_grad_enabled() and self.embedding_dim in (32, 64, 128) and self.v_feat is not None \
                and self.t_feat is not None:
            return self._forward_inference(adj)
        image_feats = ops.project(self.image_embedding.weight, self.image_trs.weight, self.image_trs.bias)
        text_feats = ops.project(self.text_embedding.weight, self.text_trs.weight, self.text_trs.bias)
        item_w = self.item_id_embedding.weight
        image_item = torch.multiply(item_w, self.gate_v(image_feats))
        text_item = torch.multiply(item_w, self.gate_t(text_feats))
        ego = torch.cat([self.user_embedding.weight, item_w], dim=0)
        content = ops.propagate_mean(adj, ego, self.n_ui_layers)
        for _ in range(self.n_layers):
            image_item = ops.spmm(self.image_original_adj, image_item)
        image_embeds = torch.cat([ops.spmm(self.R, image_item), image_item], dim=0)
        for _ in range(self.n_layers):
            text_item = ops.spmm(self.text_original_adj, text_item)
        text_embeds = torch.cat([ops.spmm(self.R, text_item), text_item], dim=0)
        att = torch.cat([self.query_common(image_embeds), self.query_common(text_embeds)], dim=-1)
        w = self.softmax(att)
        common = w[:, 0].unsqueeze(dim=1) * image_embeds + w[:, 1].unsqueeze(dim=1) * text_embeds
        sep_image, sep_text = image_embeds - common, text_embeds - common
        sep_image = torch.multiply(self.gate_image_prefer(content), sep_image)
        sep_text = torch.multiply(self.gate_text_prefer(content), sep_text)
        side = (sep_image + sep_text + common) / 3
        all_embeds = content + side
        u, i = torch.split(all_embeds, [self.n_users, self.n_items], dim=0)
        if train:
            return u, i, side, content
        return u, i

    def bpr_loss(self, users, pos_items, neg_items):
        pos = torch.sum(torch.mul(users, pos_items), dim=1)
        neg = torch.sum(torch.mul(users, neg_items), dim=1)
        reg = (1. / 2 * (users ** 2).sum() + 1. / 2 * (pos_items ** 2).sum() + 1. / 2 * (neg_items ** 2).sum()) / self.batch_size
        return -torch.mean(F.logsigmoid(pos - neg)), self.reg_weight * reg, 0.0

    def InfoNCE(self, view1, view2, temperature):
        view1, view2 = F.normalize(view1, dim=1), F.normalize(view2, dim=1)
        pos = torch.exp((view1 * view2).sum(dim=-1) / temperature)
        ttl = torch.exp(torch.matmul(view1, view2.transpose(0, 1)) / temperature).sum(dim=1)
        return torch.mean(-torch.log(pos / ttl))

    def calculate_loss(self, interaction):
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        ua, ia, side, content = self.forward(self.norm_adj, train=True)
        mf, emb, reg = self.bpr_loss(ua[users], ia[pos_items], ia[neg_items])
        side_u, side_i = torch.split(side, [self.n_users, self.n_items], dim=0)
        cont_u, cont_i = torch.split(content, [self.n_users, self.n_items], dim=0)
        cl = self.InfoNCE(side_i[pos_items], cont_i[pos_items], 0.2) + self.InfoNCE(side_u[users], cont_u[users], 0.2)
        return mf + emb + reg + self.cl_loss * cl

    def _score_embeddings(self):
        return self._cached_eval_embeddings(lambda: self.forward(self.norm_adj))

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
