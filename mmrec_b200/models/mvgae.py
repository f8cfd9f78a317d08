"""MVGAE (TMM'21) on the H100 hot path; mirrors `src/models/mvgae.py` (class names `MVGAE`, `GCN`, `ProductOfExperts`,
`BaseModel`, constructor, config keys, parameter names, registration and initialisation order: `init_seed` gives the
reference's initial weights bit for bit and a reference `state_dict` loads with `strict=True`) WITHOUT torch_geometric.

Kernels: PyG's `MessagePassing(aggr='mean')` over the symmetrised edge list with its self loops removed and added once
(`:322-329`) is the SpMM `D^-1 (A + I) (x W)` on a row-normalised CSR (`ops.spmm`); `MLP(features)` + `F.normalize` of the
item rows (`:250-254`) is `ops.project(..., l2_normalize=True)`; the hardest in-batch negative of `dot_product_decode_neg`
(`:73-85`), which the reference reaches through a [B, B, d] product (1 GiB per call at B = 2048, d = 64; four calls per
loss), is `ops.max_dot`: K3's fused score + top-1, O(B d) memory in the forward and the backward; scoring is `ops.score` /
`ops.score_topk`.  The product of experts, the KL terms, the leaky ReLUs and the small linears stay torch, called in the
reference's order.

Reference quirks kept on purpose:
- `self.dataset = 'amazon'` is hard-coded (`:32`), so `recon_loss` applies `sigmoid` to z (`:130-131`) and
  `result_embed = sigmoid(pd_mu)` (`:115-116`).
- Positive and negative item ids index z with no `+ n_users` offset (`:83`, `:88`, `:160`): they read rows of the user
  block (or item rows where an id is >= n_users).
- The decode takes the max over ALL B negatives of the batch, not over each row's own negative (`:76-84`).
- `collaborative`, each GCN's `preference` and `result_embed` are plain tensors, not Parameters (`:43`, `:58`, `:201`):
  they consume the initialisation RNG and are never trained (here they do not require grad either, so no gradient is
  computed for them).
- `full_sort_predict` scores the `result_embed` of the last forward (`:174-180`): the last training batch's forward,
  before its optimizer step; before any forward, the initial random tensor.  It is kept detached.
- Each conv's `update` applies `F.dropout(p=0.1)` in training mode (`:345`): three masks per GCN per forward, drawn in the
  order v, t, c; then `torch.randn_like` for z (`:112`) and for z_v, z_t, z_c (`:163-165`).
- `reparametrize` scales the noise by 0.1 and clamps logvar at 10 (`:66-71`, `:149`).
- `recon_loss` is a SUM of `log2` (`:135`).
- Both modalities are required: `forward` calls `v_gcn` and `t_gcn` unconditionally (`:92-93`), so construction raises
  without either feature file.
- `g_layer2` keeps torch's default initialisation (its xavier call is commented out, `:228-230`); `conv_embed_2`,
  `linear_layer2` and `g_layer2` are registered but unused at `n_layers: 1`.
Only the variants the reference runs are built: `aggr_mode = 'mean'` and `concate = False` are hard-coded (`:39-40`)."""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..common.abstract_recommender import GeneralRecommender
from .mmgcn import mean_adj_from_edges

EPS = 1e-15
MAX_LOGVAR = 10


class MVGAE(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        if self.v_feat is None or self.t_feat is None:
            # the reference's forward runs both modality towers (mvgae.py:92-93): it cannot run with one
            raise ValueError("MVGAE needs both modality feature files (image and text): "
                             f"image {'found' if self.v_feat is not None else 'missing'}, text {'found' if self.t_feat is not None else 'missing'}")
        self.experts = ProductOfExperts()
        self.dataset = "amazon"                                       # sic (mvgae.py:32)
        self.batch_size = config["train_batch_size"]
        self.num_user = self.n_users
        self.num_item = self.n_items
        num_user, num_item = self.n_users, self.n_items
        num_layer = config["n_layers"]
        self.aggr_mode = "mean"
        self.concate = False
        self.dim_x = config["embedding_size"]
        self.beta = config["beta"]
        self.collaborative = nn.init.xavier_normal_(torch.rand((num_item, self.dim_x))).to(self.device)
        inter = dataset.inter_matrix(form="coo").astype(np.float32)
        edge_index = torch.tensor(self.pack_edge_index(inter), dtype=torch.long)
        self.edge_index = edge_index.t().contiguous().to(self.device)
        self.edge_index = torch.cat((self.edge_index, self.edge_index[[1, 0]]), dim=1)
        self.mean_adj = mean_adj_from_edges(self.edge_index, num_user + num_item, self_loops=True)
        args = (self.device, self.edge_index, self.batch_size, num_user, num_item, self.dim_x, self.aggr_mode, self.concate)
        self.v_gcn = GCN(args[0], self.v_feat, *args[1:], num_layer=num_layer, dim_latent=128, mean_adj=self.mean_adj)
        self.t_gcn = GCN(args[0], self.t_feat, *args[1:], num_layer=num_layer, dim_latent=128, mean_adj=self.mean_adj)
        self.c_gcn = GCN(args[0], self.collaborative, *args[1:], num_layer=num_layer, dim_latent=128, mean_adj=self.mean_adj)
        self.result_embed = nn.init.xavier_normal_(torch.rand((num_user + num_item, self.dim_x))).to(self.device)

    def pack_edge_index(self, inter_mat):
        return np.column_stack((inter_mat.row, inter_mat.col + self.n_users))

    def reparametrize(self, mu, logvar):
        logvar = logvar.clamp(max=MAX_LOGVAR)
        if self.training:
            return mu + torch.randn_like(logvar) * 0.1 * torch.exp(logvar.mul(0.5))
        return mu

    def dot_product_decode_neg(self, z, user, neg_items, sigmoid=True):
        max_neg_value, _ = ops.max_dot(z[user], z[neg_items])            # K3 top-1: no [B, B, d] tensor
        return torch.sigmoid(max_neg_value) if sigmoid else max_neg_value

    def dot_product_decode(self, z, edge_index, sigmoid=True):
        value = torch.sum(z[edge_index[0]] * z[edge_index[1]], dim=1)
        return torch.sigmoid(value) if sigmoid else value

    def forward(self):
        v_mu, v_logvar = self.v_gcn()
        t_mu, t_logvar = self.t_gcn()
        c_mu, c_logvar = self.c_gcn()
        self.v_logvar, self.t_logvar, self.v_mu, self.t_mu = v_logvar, t_logvar, v_mu, t_mu
        pd_mu, pd_logvar, _ = self.experts(torch.stack([v_mu, t_mu], dim=0), torch.stack([v_logvar, t_logvar], dim=0))
        pd_mu, pd_logvar, _ = self.experts(torch.stack([pd_mu, c_mu], dim=0), torch.stack([pd_logvar, c_logvar], dim=0))
        z = self.reparametrize(pd_mu, pd_logvar)
        self.result_embed = torch.sigmoid(pd_mu).detach()            # 'amazon' (mvgae.py:115-116); scored by full_sort_predict
        return pd_mu, pd_logvar, z, v_mu, v_logvar, t_mu, t_logvar, c_mu, c_logvar

    def recon_loss(self, z, pos_edge_index, user, neg_items):
        z = torch.sigmoid(z)                                          # 'amazon' (mvgae.py:130-131)
        pos_scores = self.dot_product_decode(z, pos_edge_index, sigmoid=True)
        neg_scores = self.dot_product_decode_neg(z, user, neg_items, sigmoid=True)
        return -torch.sum(torch.log2(torch.sigmoid(pos_scores - neg_scores)))

    def kl_loss(self, mu, logvar):
        logvar = logvar.clamp(max=MAX_LOGVAR)
        return -0.5 * torch.mean(torch.sum(1 + logvar - mu ** 2 - logvar.exp(), dim=1))

    def calculate_loss(self, interaction):
        user, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        pos_edge_index = torch.stack([user, pos_items], dim=0)
        pd_mu, pd_logvar, z, v_mu, v_logvar, t_mu, t_logvar, c_mu, c_logvar = self.forward()
        z_v = self.reparametrize(v_mu, v_logvar)
        z_t = self.reparametrize(t_mu, t_logvar)
        z_c = self.reparametrize(c_mu, c_logvar)
        recon_loss = self.recon_loss(z, pos_edge_index, user, neg_items)
        kl_loss = self.kl_loss(pd_mu, pd_logvar)
        loss_multi = recon_loss + self.beta * kl_loss
        loss_v = self.recon_loss(z_v, pos_edge_index, user, neg_items) + self.beta * self.kl_loss(v_mu, v_logvar)
        loss_t = self.recon_loss(z_t, pos_edge_index, user, neg_items) + self.beta * self.kl_loss(t_mu, t_logvar)
        loss_c = self.recon_loss(z_c, pos_edge_index, user, neg_items) + self.beta * self.kl_loss(c_mu, c_logvar)
        return loss_multi + loss_v + loss_t + loss_c

    def _score_embeddings(self):
        res = self.result_embed.detach()
        return res[:self.n_users].contiguous(), res[self.n_users:].contiguous()

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])


class GCN(nn.Module):
    """`mvgae.py:183-282`, the `concate = False` path."""

    def __init__(self, device, features, edge_index, batch_size, num_user, num_item, dim_id, aggr_mode, concate,
                 num_layer, dim_latent=None, mean_adj=None):
        super().__init__()
        self.device = device
        self.batch_size = batch_size
        self.num_user = num_user
        self.num_item = num_item
        self.dim_id = dim_id
        self.dim_feat = features.size(1)
        self.dim_latent = dim_latent
        self.edge_index = edge_index
        self.features = features
        self.aggr_mode = aggr_mode
        self.concate = concate
        self.num_layer = num_layer
        self.mean_adj = mean_adj
        if concate:
            raise NotImplementedError("MVGAE's GCN: only the concate = False path the reference runs (mvgae.py:40)")
        d_in = self.dim_latent if self.dim_latent else self.dim_feat
        self.preference = nn.init.xavier_normal_(torch.rand((num_user, d_in))).to(self.device)
        if self.dim_latent:
            self.MLP = nn.Linear(self.dim_feat, self.dim_latent)
            nn.init.xavier_normal_(self.MLP.weight)
        self.conv_embed_1 = BaseModel(d_in, self.dim_id, aggr=self.aggr_mode)
        nn.init.xavier_normal_(self.conv_embed_1.weight)
        self.linear_layer1 = nn.Linear(d_in, self.dim_id)
        nn.init.xavier_normal_(self.linear_layer1.weight)
        self.g_layer1 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.g_layer1.weight)
        self.conv_embed_2 = BaseModel(self.dim_id, self.dim_id, aggr=self.aggr_mode)
        nn.init.xavier_normal_(self.conv_embed_2.weight)
        self.linear_layer2 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.linear_layer2.weight)
        self.g_layer2 = nn.Linear(self.dim_id, self.dim_id)           # sic: no xavier init (mvgae.py:230)
        self.conv_embed_4 = BaseModel(self.dim_id, self.dim_id, aggr=self.aggr_mode)
        nn.init.xavier_normal_(self.conv_embed_4.weight)
        self.linear_layer4 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.linear_layer4.weight)
        self.g_layer4 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.g_layer4.weight)
        self.conv_embed_5 = BaseModel(self.dim_id, self.dim_id, aggr=self.aggr_mode)
        nn.init.xavier_normal_(self.conv_embed_5.weight)
        self.linear_layer5 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.linear_layer5.weight)
        self.g_layer5 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.g_layer5.weight)

    def forward(self):
        if self.dim_latent:   # item rows: gather-free linear + L2 normalise in one kernel (normalising the cat is row-wise)
            items = ops.project(self.features, self.MLP.weight, self.MLP.bias, l2_normalize=True)
        else:
            items = F.normalize(self.features)
        x = torch.cat((F.normalize(self.preference), items), dim=0)
        # (the reference also computes leaky_relu(linear_layer1/2(x)) here and discards it when concate is False)
        if self.num_layer > 0:
            x = F.leaky_relu(self.g_layer1(F.leaky_relu(self.conv_embed_1(x, self.mean_adj))))
        if self.num_layer > 1:
            x = F.leaky_relu(self.g_layer2(F.leaky_relu(self.conv_embed_2(x, self.mean_adj))))
        mu = F.leaky_relu(self.conv_embed_4(x, self.mean_adj))
        mu = self.g_layer4(mu) + F.leaky_relu(self.linear_layer4(x))
        logvar = F.leaky_relu(self.conv_embed_5(x, self.mean_adj))
        logvar = self.g_layer5(logvar) + F.leaky_relu(self.linear_layer5(x))
        return mu, logvar


class ProductOfExperts(nn.Module):
    """`mvgae.py:285-301`: precision-weighted mean of M Gaussian experts."""

    def forward(self, mu, logvar, eps=1e-8):
        var = torch.exp(logvar) + eps
        T = 1. / var
        pd_mu = torch.sum(mu * T, dim=0) / torch.sum(T, dim=0)
        pd_var = 1. / torch.sum(T, dim=0)
        pd_logvar = torch.log(pd_var)
        return pd_mu, pd_logvar, pd_var


class BaseModel(nn.Module):
    """`mvgae.py:304-345`: x @ weight, mean over the in-neighbours and the node itself (K1), + bias, L2 normalise, dropout."""

    def __init__(self, in_channels, out_channels, normalize=True, bias=True, aggr="add", **kwargs):
        super().__init__()
        self.aggr = aggr
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.normalize = normalize
        self.weight = nn.Parameter(torch.Tensor(self.in_channels, out_channels))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.in_channels)                    # torch_geometric.nn.inits.uniform
        self.weight.data.uniform_(-bound, bound)
        if self.bias is not None:
            self.bias.data.uniform_(-bound, bound)

    def forward(self, x, mean_adj, size=None):
        return self.update(ops.spmm(mean_adj, torch.matmul(x, self.weight)))

    def update(self, aggr_out):
        if self.bias is not None:
            aggr_out = aggr_out + self.bias
        if self.normalize:
            aggr_out = F.normalize(aggr_out, p=2, dim=-1)
        return F.dropout(aggr_out, p=0.1, training=self.training)
