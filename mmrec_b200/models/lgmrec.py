"""LGMRec on the H100 hot path; mirrors `src/models/lgmrec.py` (class name, config keys, parameter names, registration and
initialisation order).  LightGCN propagation (`:89-100`, `:111-112`) -> ops.propagate_mean / ops.spmm on CSR; the four
whole-table products of each frozen feature table (`:105-107`, `:118`, `:123`) -> ONE ops.project per table with
`[trs | hyper]` concatenated; `torch.sparse.mm` on R (`:108`, `:119`, `:124`) -> ops.spmm; the full-table exp-sums of the
hypergraph contrastive loss (`:164`) -> ops.expsum_rows (K8); scoring (`:196-200`) -> ops.score.  The Gumbel softmax, the
dropouts, the [H, d] hypergraph layer and the combine stay torch on the device, called in the reference's order.

The reference draws random numbers in EVERY forward, evaluation included (`F.gumbel_softmax`, `:120-126`), so no
embeddings are cached across `full_sort_predict` / `full_sort_topk` calls: each runs its own forward, as the reference's
does."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from ..common.abstract_recommender import GeneralRecommender


class LGMRec(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.embedding_dim = config["embedding_size"]
        self.feat_embed_dim = config["feat_embed_dim"]
        self.cf_model = config["cf_model"]
        self.n_mm_layer = config["n_mm_layers"]
        self.n_ui_layers = config["n_ui_layers"]
        self.n_hyper_layer = config["n_hyper_layer"]
        self.hyper_num = config["hyper_num"]
        self.keep_rate = config["keep_rate"]
        self.alpha = config["alpha"]
        self.cl_weight = config["cl_weight"]
        self.reg_weight = config["reg_weight"]
        self.tau = 0.2
        self.n_nodes = self.n_users + self.n_items
        if self.v_feat is None or self.t_feat is None:
            # the reference's forward reads the hyperedge embeddings of both modalities (lgmrec.py:151): it cannot run with one
            raise ValueError("LGMRec needs both modality feature files (image and text): "
                             f"image {'found' if self.v_feat is not None else 'missing'}, text {'found' if self.t_feat is not None else 'missing'}")
        self.hgnnLayer = HGNNLayer(self.n_hyper_layer)

        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        inter = self.interaction_matrix
        self.adj = ops.CSR.from_coo(torch.from_numpy(inter.row.astype(np.int64)).to(self.device),
                                    torch.from_numpy(inter.col.astype(np.int64)).to(self.device),
                                    torch.from_numpy(inter.data.astype(np.float32)).to(self.device), self.n_users, self.n_items)
        self.norm_adj = graph.build_norm_adj(inter, self.n_users, self.n_items, self.device)
        # lgmrec.py:78 + :43: degree of the binary symmetric matrix, 1 / (deg + 1e-7) in float64, then fp32; [N, 1]
        rows, _, n = graph._sym_keys(inter.row, inter.col, self.n_users, self.n_items)
        deg = np.bincount(rows, minlength=n).astype(np.float64).reshape(-1, 1)
        self.num_inters = torch.from_numpy((1.0 / (deg + 1e-7)).astype(np.float32)).to(self.device)

        self.user_embedding = nn.Embedding(self.n_users, self.embedding_dim)
        self.item_id_embedding = nn.Embedding(self.n_items, self.embedding_dim)
        nn.init.xavier_uniform_(self.user_embedding.weight)
        nn.init.xavier_uniform_(self.item_id_embedding.weight)
        self.drop = nn.Dropout(p=1 - self.keep_rate)
        self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=True)
        self.item_image_trs = nn.Parameter(nn.init.xavier_uniform_(torch.zeros(self.v_feat.shape[1], self.feat_embed_dim)))
        self.v_hyper = nn.Parameter(nn.init.xavier_uniform_(torch.zeros(self.v_feat.shape[1], self.hyper_num)))
        self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=True)
        self.item_text_trs = nn.Parameter(nn.init.xavier_uniform_(torch.zeros(self.t_feat.shape[1], self.feat_embed_dim)))
        self.t_hyper = nn.Parameter(nn.init.xavier_uniform_(torch.zeros(self.t_feat.shape[1], self.hyper_num)))

    def _project(self, table, trs, hyper):
        """(table @ trs, table @ hyper) in one pass over the frozen table: K2 with the two weights side by side, the width
        padded with zero columns to a multiple of 64 (the tile width of its tensor-core path: 128 for H = 4 or 64).  The
        backward is K5's weight gradient over the whole table; the table has none."""
        d, H = trs.shape[1], hyper.shape[1]
        pad = -(d + H) % 64
        parts = [trs, hyper] + ([trs.new_zeros(trs.shape[0], pad)] if pad else [])
        y = ops.project(table, torch.cat(parts, dim=1).t())
        return y[:, :d], y[:, d:d + H]

    def cge(self):
        ego = torch.cat((self.user_embedding.weight, self.item_id_embedding.weight), dim=0)
        if self.cf_model == "mf":
            return ego
        if self.cf_model == "lightgcn":
            return ops.propagate_mean(self.norm_adj, ego, self.n_ui_layers)

    def mge(self, item_feats):
        user_feats = ops.spmm(self.adj, item_feats) * self.num_inters[:self.n_users]
        mge_feats = torch.cat([user_feats, item_feats], dim=0)
        for _ in range(self.n_mm_layer):
            mge_feats = ops.spmm(self.norm_adj, mge_feats)
        return mge_feats

    def forward(self):
        v_item, iv_hyper = self._project(self.image_embedding.weight, self.item_image_trs, self.v_hyper)
        uv_hyper = ops.spmm(self.adj, iv_hyper)
        iv_hyper = F.gumbel_softmax(iv_hyper, self.tau, dim=1, hard=False)
        uv_hyper = F.gumbel_softmax(uv_hyper, self.tau, dim=1, hard=False)
        t_item, it_hyper = self._project(self.text_embedding.weight, self.item_text_trs, self.t_hyper)
        ut_hyper = ops.spmm(self.adj, it_hyper)
        it_hyper = F.gumbel_softmax(it_hyper, self.tau, dim=1, hard=False)
        ut_hyper = F.gumbel_softmax(ut_hyper, self.tau, dim=1, hard=False)

        cge_embs = self.cge()
        v_feats = self.mge(v_item)
        t_feats = self.mge(t_item)
        mge_embs = F.normalize(v_feats) + F.normalize(t_feats)
        lge_embs = cge_embs + mge_embs
        uv_hyper_embs, iv_hyper_embs = self.hgnnLayer(self.drop(iv_hyper), self.drop(uv_hyper), cge_embs[self.n_users:])
        ut_hyper_embs, it_hyper_embs = self.hgnnLayer(self.drop(it_hyper), self.drop(ut_hyper), cge_embs[self.n_users:])
        av_hyper_embs = torch.concat([uv_hyper_embs, iv_hyper_embs], dim=0)
        at_hyper_embs = torch.concat([ut_hyper_embs, it_hyper_embs], dim=0)
        ghe_embs = av_hyper_embs + at_hyper_embs
        all_embs = lge_embs + self.alpha * F.normalize(ghe_embs)
        u_embs, i_embs = torch.split(all_embs, [self.n_users, self.n_items], dim=0)
        return u_embs, i_embs, [uv_hyper_embs, iv_hyper_embs, ut_hyper_embs, it_hyper_embs]

    def bpr_loss(self, users, pos_items, neg_items):
        pos_scores = torch.sum(torch.mul(users, pos_items), dim=1)
        neg_scores = torch.sum(torch.mul(users, neg_items), dim=1)
        return -torch.mean(F.logsigmoid(pos_scores - neg_scores))

    def ssl_triple_loss(self, emb1, emb2, all_emb):
        norm_emb1 = F.normalize(emb1)
        norm_emb2 = F.normalize(emb2)
        norm_all_emb = F.normalize(all_emb)
        pos_score = torch.exp(torch.mul(norm_emb1, norm_emb2).sum(dim=1) / self.tau)
        ttl_score = ops.expsum_rows(norm_emb1, norm_all_emb, self.tau)        # K8: no [B, M] matrix
        return -torch.log(pos_score / ttl_score).sum()

    def reg_loss(self, *embs):
        reg_loss = 0
        for emb in embs:
            reg_loss += torch.norm(emb, p=2)
        reg_loss /= embs[-1].shape[0]
        return reg_loss

    def calculate_loss(self, interaction):
        ua_embeddings, ia_embeddings, hyper_embeddings = self.forward()
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        u_g_embeddings = ua_embeddings[users]
        pos_i_g_embeddings = ia_embeddings[pos_items]
        neg_i_g_embeddings = ia_embeddings[neg_items]
        batch_bpr_loss = self.bpr_loss(u_g_embeddings, pos_i_g_embeddings, neg_i_g_embeddings)
        uv_embs, iv_embs, ut_embs, it_embs = hyper_embeddings
        batch_hcl_loss = self.ssl_triple_loss(uv_embs[users], ut_embs[users], ut_embs) + \
            self.ssl_triple_loss(iv_embs[pos_items], it_embs[pos_items], it_embs)
        batch_reg_loss = self.reg_loss(u_g_embeddings, pos_i_g_embeddings, neg_i_g_embeddings)
        return batch_bpr_loss + self.cl_weight * batch_hcl_loss + self.reg_weight * batch_reg_loss

    def _score_embeddings(self):
        u, i, _ = self.forward()                                    # a fresh forward per call (its Gumbel draws), never cached
        return u, i

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])


class HGNNLayer(nn.Module):
    def __init__(self, n_hyper_layer):
        super().__init__()
        self.h_layer = n_hyper_layer

    def forward(self, i_hyper, u_hyper, embeds):
        i_ret = embeds
        for _ in range(self.h_layer):
            lat = torch.mm(i_hyper.T, i_ret)
            i_ret = torch.mm(i_hyper, lat)
            u_ret = torch.mm(u_hyper, lat)
        return u_ret, i_ret
