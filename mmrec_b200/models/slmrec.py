"""SLMRec (TMM'22) on the H100 hot path; mirrors `src/models/slmrec.py` (class name, constructor, config keys, module and
parameter names, registration and initialisation order: `init_seed` gives the reference's initial state bit for bit).

Kernels: `compute()` (`:73-118`) runs three LightGCN propagations of one adjacency -- the id view `[E_u; E_i]`, the visual
view `[E_u; v_dense(v_feat)]` and the text view `[E_u; t_dense(t_feat)]` -- and feeds the column concatenation `[id | v | t]`
of their outputs to `embedding_{user,item}_after_GCN`.  A column block of `A [X1 | X2 | X3]` is `A Xk`, so here it is ONE
propagation of the [N, 3d] ego table `[[E_u, E_u, E_u]; [E_i, V, T]]` (`ops.propagate_mean`: K1 at width 3d, one SpMM per
layer instead of three; each d-wide block is bit-identical to the width-d propagation of that view).  Its user and item rows
are the concat-fused tables; the `i_emb_*`, `v_emb_*`, `t_emb_*` views that FAC reads are column-block views of them.  The
projections `v_dense` / `t_dense` of the L2-normalised frozen tables run on K2 (`ops.project`); the adjacency is
`graph.build_slmrec_adj` for every `adj_type`.  The two linears, `infonce` and the FAC heads stay torch, in the reference's
order.

Reference semantics kept on purpose:
- `full_sort_predict` scores the `all_users` / `all_items` stored by the LAST `calculate_loss` (`:307-318`), computed
  before that step's optimiser update; it does not recompute them, so evaluating before any training batch fails.
- It returns `sigmoid(scores)` (`:315`).  `full_sort_topk` therefore ranks the sigmoid of the scores (`ops.score`, in-place
  sigmoid, `ops.mask_topk`), not the raw scores of the fused top-k: in fp32, sigmoid maps distinct large scores to equal
  values, whose ties go to the lower item index, as `torch.topk` of the masked `full_sort_predict` does.
- Only what the reference can run is built.  These raise `MMRecError` at construction: `ssl_task` other than `FAC` (`FD` /
  `FM` read `self.a_dense_emb`, which never exists), `mm_fusion_mode: mean` (the linears expect width 3d), `init: normal`
  (it reads `embedding_item_ID`), and a missing image or text table or `dataset: kwai` (its two-view branch is not built).
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from .._lib import MMRecError
from ..common.abstract_recommender import GeneralRecommender


class SLMRec(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self._check_supported(config)
        self.a_feat = None
        self.config = config
        self.infonce_criterion = nn.CrossEntropyLoss()
        self.num_users = self.n_users
        self.num_items = self.n_items
        self.latent_dim = config["recdim"]
        self.n_layers = config["layer_num"]
        self.mm_fusion_mode = config["mm_fusion_mode"]
        self.temp = config["temp"]
        self.create_u_embeding_i()
        self.all_items = self.all_users = None
        inter = dataset.inter_matrix(form="coo")
        self.norm_adj = graph.build_slmrec_adj(inter, self.n_users, self.n_items, self.device, config["adj_type"])
        self.f = nn.Sigmoid()
        d = self.latent_dim
        self.g_i_iv = nn.Linear(d, d)
        self.g_v_iv = nn.Linear(d, d)
        self.g_iv_iva = nn.Linear(d, d)
        self.g_a_iva = nn.Linear(d, d)
        self.g_iva_ivat = nn.Linear(d, d // 2)
        self.g_t_ivat = nn.Linear(d, d // 2)
        for m in (self.g_i_iv, self.g_v_iv, self.g_iv_iva, self.g_a_iva, self.g_iva_ivat, self.g_t_ivat):
            nn.init.xavier_uniform_(m.weight)
        self.ssl_temp = config["ssl_temp"]

    def _check_supported(self, config):
        why = []
        if config["ssl_task"] != "FAC":
            why.append(f"ssl_task {config['ssl_task']!r}: only 'FAC' runs in the reference (FD / FM read a_dense_emb, never built)")
        if config["mm_fusion_mode"] != "concat":
            why.append(f"mm_fusion_mode {config['mm_fusion_mode']!r}: the after-GCN linears expect the width-3d concatenation")
        if config["init"] == "normal":
            why.append("init 'normal': the reference reads embedding_item_ID, which does not exist")
        if self.v_feat is None or self.t_feat is None or config["dataset"] == "kwai":
            why.append("SLMRec is built for the three views id, image and text: both feature tables are required "
                       f"(image {'found' if self.v_feat is not None else 'missing'}, text {'found' if self.t_feat is not None else 'missing'}, "
                       f"dataset {config['dataset']!r}; the two-view 'kwai' branch is not built)")
        if why:
            raise MMRecError("SLMRec: unsupported configuration: " + "; ".join(why))

    def create_u_embeding_i(self):
        self.embedding_user = nn.Embedding(num_embeddings=self.num_users, embedding_dim=self.latent_dim)
        self.embedding_item = nn.Embedding(num_embeddings=self.num_items, embedding_dim=self.latent_dim)
        if self.config["init"] == "xavier":
            nn.init.xavier_uniform_(self.embedding_user.weight, gain=1)
            nn.init.xavier_uniform_(self.embedding_item.weight, gain=1)
        self.v_feat = F.normalize(self.v_feat, dim=1)
        self.v_dense = nn.Linear(self.v_feat.shape[1], self.latent_dim)
        nn.init.xavier_uniform_(self.v_dense.weight)
        self.t_feat = F.normalize(self.t_feat, dim=1)
        self.t_dense = nn.Linear(self.t_feat.shape[1], self.latent_dim)
        nn.init.xavier_uniform_(self.t_dense.weight)
        self.item_feat_dim = self.latent_dim * 3
        self.embedding_item_after_GCN = nn.Linear(self.item_feat_dim, self.latent_dim)
        self.embedding_user_after_GCN = nn.Linear(self.item_feat_dim, self.latent_dim)
        nn.init.xavier_uniform_(self.embedding_item_after_GCN.weight)
        nn.init.xavier_uniform_(self.embedding_user_after_GCN.weight)

    def compute(self):
        users_emb = self.embedding_user.weight
        items_emb = self.embedding_item.weight
        self.v_dense_emb = ops.project(self.v_feat, self.v_dense.weight, self.v_dense.bias)
        self.t_dense_emb = ops.project(self.t_feat, self.t_dense.weight, self.t_dense.bias)
        ego = torch.cat([torch.cat([users_emb, users_emb, users_emb], dim=1),
                         torch.cat([items_emb, self.v_dense_emb, self.t_dense_emb], dim=1)])
        out = ops.propagate_mean(self.norm_adj, ego, self.n_layers)    # [N, 3d]: the id, image and text views side by side
        d, nu = self.latent_dim, self.num_users
        self.i_emb, self.v_emb, self.t_emb = out[:, :d], out[:, d:2 * d], out[:, 2 * d:]
        self.i_emb_u, self.i_emb_i = self.i_emb[:nu], self.i_emb[nu:]
        self.v_emb_u, self.v_emb_i = self.v_emb[:nu], self.v_emb[nu:]
        self.t_emb_u, self.t_emb_i = self.t_emb[:nu], self.t_emb[nu:]
        user = self.embedding_user_after_GCN(out[:nu])                  # = mm_fusion([i_emb_u, v_emb_u, t_emb_u]), 'concat'
        item = self.embedding_item_after_GCN(out[nu:])
        return user, item

    def fac(self, idx):
        x_i_iv = self.g_i_iv(self.i_emb_i[idx])
        x_v_iv = self.g_v_iv(self.v_emb_i[idx])
        v_logits = torch.mm(x_i_iv, x_v_iv.T)
        v_logits /= self.ssl_temp
        v_labels = torch.arange(x_i_iv.shape[0], device=v_logits.device)
        v_loss = self.infonce_criterion(v_logits, v_labels)
        x_iv_iva = self.g_iv_iva(x_i_iv)
        x_iva_ivat = self.g_iva_ivat(x_iv_iva)
        x_t_ivat = self.g_t_ivat(self.t_emb_i[idx])
        t_logits = torch.mm(x_iva_ivat, x_t_ivat.T)
        t_logits /= self.ssl_temp
        t_labels = torch.arange(x_iva_ivat.shape[0], device=t_logits.device)
        t_loss = self.infonce_criterion(t_logits, t_labels)
        return v_loss + t_loss

    def _stored_tables(self, candidate_items=None):
        if self.all_users is None:
            raise MMRecError("SLMRec scores the tables stored by the last calculate_loss: run a training batch first")
        items = self.all_items
        if candidate_items is not None:
            items = items[torch.as_tensor(candidate_items, device=items.device).long()]
        return self.all_users.detach(), items.detach()

    def full_sort_predict(self, interaction, candidate_items=None):
        u, i = self._stored_tables(candidate_items)
        return torch.sigmoid_(ops.score(u, i, interaction[0]))

    def full_sort_topk(self, interaction, k):
        """`full_sort_predict` + `scores[mask] = -1e10` + `torch.topk` on the sigmoid scores (see the module docstring)."""
        u, i = self._stored_tables()
        scores = torch.sigmoid_(ops.score(u, i, interaction[0]))
        _, idx = ops.mask_topk(scores, interaction[1], k)
        return idx

    def getEmbedding(self, users, pos_items, neg_items):
        self.all_users, self.all_items = self.compute()
        users_emb = self.all_users[users]
        pos_emb = self.all_items[pos_items]
        users_emb_ego = self.embedding_user(users)
        pos_emb_ego = self.embedding_item(pos_items)
        if neg_items is None:
            neg_emb_ego = neg_emb = None
        else:
            neg_emb = self.all_items[neg_items]
            neg_emb_ego = self.embedding_item(neg_items)
        return users_emb, pos_emb, neg_emb, users_emb_ego, pos_emb_ego, neg_emb_ego

    def calculate_loss(self, interaction):
        users, pos = interaction[0], interaction[1]
        main_loss = self.infonce(users, pos)
        ssl_loss = self.compute_ssl(users, pos)
        return main_loss + self.config["ssl_alpha"] * ssl_loss

    def ssl_loss(self, users, pos):
        self.getEmbedding(users.long(), pos.long(), None)
        return self.compute_ssl(users, pos)

    def compute_ssl(self, users, items):
        return self.fac(items)

    def forward(self, users, items):
        all_users, all_items = self.compute()
        gamma = torch.sum(torch.mul(all_users[users], all_items[items]), dim=1)
        return gamma.detach()

    def infonce(self, users, pos):
        users_emb, pos_emb = self.getEmbedding(users.long(), pos.long(), None)[:2]
        users_emb = F.normalize(users_emb, dim=1)
        pos_emb = F.normalize(pos_emb, dim=1)
        logits = torch.mm(users_emb, pos_emb.T)
        logits /= self.temp
        labels = torch.arange(users_emb.shape[0], device=logits.device)
        return self.infonce_criterion(logits, labels)
