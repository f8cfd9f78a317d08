"""MMGCN on the H100 hot path; mirrors `src/models/mmgcn.py` (class names, constructor, attribute and
parameter names, registration order) WITHOUT torch_geometric: PyG's `MessagePassing(aggr='mean')` with
`message = x_j` (`mmgcn.py:191-213`) over the symmetrised edge list (`:40-42`) is the SpMM `D^-1 A (x W)`, run by
`ops.spmm` on a row-normalised CSR; `MLP(features)` + `F.normalize` (`:165-168`) for the item rows is the fused
gather -> linear -> L2-normalise kernel `ops.project(..., l2_normalize=True)`.

Parity: torch_geometric is not a dependency; the reference's file was run under a shim of its one PyG primitive
(tests/golden/ref_loader.py) to record tests/golden/mmgcn_tiny.npz, and the kernels are checked against `oracle.mmgcn_*` (pinned to the same file) in tests/test_gpu_models.py.  Unpinned: the mean aggregation
primitive itself (shim and oracle restate PyG's documented formula).  Reference quirks kept on purpose: `concate = 'False'` is a non-empty string and
therefore truthy, so the concatenating variant of every layer is the one that runs (`:31,129-137,171-172`);
`preference`, `id_embedding` and `result` are plain tensors, not Parameters (`:55-56,127`), so the optimiser never
updates them; `full_sort_predict` scores the `result` cached by the last `forward` (`:99-105`).
"""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..common.abstract_recommender import GeneralRecommender
from ..ops import CSR


def mean_adj_from_edges(edge_index: torch.Tensor, n_nodes: int) -> CSR:
    """Row-normalised adjacency of PyG's mean aggregation: out[dst] = mean over edges (src -> dst) of x[src]."""
    src, dst = edge_index[0], edge_index[1]
    deg = torch.zeros(n_nodes, dtype=torch.float32, device=src.device).index_add_(0, dst, torch.ones_like(dst, dtype=torch.float32))
    vals = 1.0 / deg[dst]
    return CSR.from_coo(dst, src, vals, n_nodes, n_nodes, sum_duplicates=True, symmetric=False)


class BaseModel(nn.Module):
    """`mmgcn.py:191-213`: x @ weight, then mean over the in-neighbours."""

    def __init__(self, in_channels, out_channels, normalize=True, bias=True, aggr="add", **kwargs):
        super().__init__()
        self.aggr, self.in_channels, self.out_channels, self.normalize = aggr, in_channels, out_channels, normalize
        self.weight = nn.Parameter(torch.Tensor(self.in_channels, out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        bound = 1.0 / math.sqrt(self.in_channels)           # torch_geometric.nn.inits.uniform
        self.weight.data.uniform_(-bound, bound)

    def forward(self, x, mean_adj: CSR, size=None):
        return ops.spmm(mean_adj, torch.matmul(x, self.weight))


class GCN(nn.Module):
    """`mmgcn.py:108-188`."""

    def __init__(self, edge_index, batch_size, num_user, num_item, dim_feat, dim_id, aggr_mode, concate, num_layer, has_id,
                 dim_latent=None, device="cpu", mean_adj=None):
        super().__init__()
        self.batch_size, self.num_user, self.num_item = batch_size, num_user, num_item
        self.dim_id, self.dim_feat, self.dim_latent = dim_id, dim_feat, dim_latent
        self.edge_index, self.aggr_mode, self.concate, self.num_layer, self.has_id, self.device = \
            edge_index, aggr_mode, concate, num_layer, has_id, device
        self.mean_adj = mean_adj
        d_in = self.dim_latent if self.dim_latent else self.dim_feat
        self.preference = nn.init.xavier_normal_(torch.rand((num_user, d_in), requires_grad=True)).to(self.device)
        if self.dim_latent:
            self.MLP = nn.Linear(self.dim_feat, self.dim_latent)
        self.conv_embed_1 = BaseModel(d_in, d_in, aggr=self.aggr_mode)
        nn.init.xavier_normal_(self.conv_embed_1.weight)
        self.linear_layer1 = nn.Linear(d_in, self.dim_id)
        nn.init.xavier_normal_(self.linear_layer1.weight)
        self.g_layer1 = nn.Linear(d_in + self.dim_id, self.dim_id) if self.concate else nn.Linear(d_in, self.dim_id)
        nn.init.xavier_normal_(self.g_layer1.weight)
        self.conv_embed_2 = BaseModel(self.dim_id, self.dim_id, aggr=self.aggr_mode)
        nn.init.xavier_normal_(self.conv_embed_2.weight)
        self.linear_layer2 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.linear_layer2.weight)
        self.g_layer2 = nn.Linear(self.dim_id + self.dim_id, self.dim_id) if self.concate else nn.Linear(self.dim_id, self.dim_id)
        self.conv_embed_3 = BaseModel(self.dim_id, self.dim_id, aggr=self.aggr_mode)
        nn.init.xavier_normal_(self.conv_embed_3.weight)
        self.linear_layer3 = nn.Linear(self.dim_id, self.dim_id)
        nn.init.xavier_normal_(self.linear_layer3.weight)
        self.g_layer3 = nn.Linear(self.dim_id + self.dim_id, self.dim_id) if self.concate else nn.Linear(self.dim_id, self.dim_id)

    def _layer(self, x, id_embedding, conv, lin, g):
        h = F.leaky_relu(conv(x, self.mean_adj))
        x_hat = F.leaky_relu(lin(x)) + id_embedding if self.has_id else F.leaky_relu(lin(x))
        return F.leaky_relu(g(torch.cat((h, x_hat), dim=1))) if self.concate else F.leaky_relu(g(h) + x_hat)

    def forward(self, features, id_embedding):
        pref = self.preference.to(features.device)
        if self.dim_latent:   # fused gather -> linear -> L2 normalise for the item rows (row-wise op: == normalising the cat)
            items = ops.project(features, self.MLP.weight, self.MLP.bias, l2_normalize=True)
        else:
            items = F.normalize(features)
        x = torch.cat((F.normalize(pref), items), dim=0)
        x = self._layer(x, id_embedding, self.conv_embed_1, self.linear_layer1, self.g_layer1)
        x = self._layer(x, id_embedding, self.conv_embed_2, self.linear_layer2, self.g_layer2)
        x = self._layer(x, id_embedding, self.conv_embed_3, self.linear_layer3, self.g_layer3)
        return x


class MMGCN(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.num_user, self.num_item = self.n_users, self.n_items
        dim_x = config["embedding_size"]
        num_layer = config["n_layers"]
        batch_size = config["train_batch_size"]
        self.aggr_mode = "mean"
        self.concate = "False"                               # sic: truthy string (mmgcn.py:31)
        has_id = True
        self.weight = torch.tensor([[1.0], [-1.0]]).to(self.device)
        self.reg_weight = config["reg_weight"]
        inter = dataset.inter_matrix(form="coo").astype(np.float32)
        edge = torch.tensor(np.column_stack((inter.row, inter.col + self.n_users)), dtype=torch.long)
        self.edge_index = edge.t().contiguous().to(self.device)
        self.edge_index = torch.cat((self.edge_index, self.edge_index[[1, 0]]), dim=1)
        self.mean_adj = mean_adj_from_edges(self.edge_index, self.n_users + self.n_items)
        self.num_modal = 0
        if self.v_feat is not None:
            self.v_gcn = GCN(self.edge_index, batch_size, self.num_user, self.num_item, self.v_feat.size(1), dim_x, self.aggr_mode,
                             self.concate, num_layer=num_layer, has_id=has_id, dim_latent=256, device=self.device,
                             mean_adj=self.mean_adj)
            self.num_modal += 1
        if self.t_feat is not None:
            self.t_gcn = GCN(self.edge_index, batch_size, self.num_user, self.num_item, self.t_feat.size(1), dim_x, self.aggr_mode,
                             self.concate, num_layer=num_layer, has_id=has_id, device=self.device, mean_adj=self.mean_adj)
            self.num_modal += 1
        self.id_embedding = nn.init.xavier_normal_(torch.rand((self.num_user + self.num_item, dim_x), requires_grad=True)).to(self.device)
        self.result = nn.init.xavier_normal_(torch.rand((self.num_user + self.num_item, dim_x))).to(self.device)

    def forward(self):
        rep = None
        if self.v_feat is not None:
            rep = self.v_gcn(self.v_feat, self.id_embedding)
        if self.t_feat is not None:
            rep = self.t_gcn(self.t_feat, self.id_embedding) if rep is None else rep + self.t_gcn(self.t_feat, self.id_embedding)
        rep = rep / self.num_modal
        self.result = rep
        return rep

    def calculate_loss(self, interaction):
        batch_users = interaction[0]
        pos_items = interaction[1] + self.n_users
        neg_items = interaction[2] + self.n_users
        user_tensor = batch_users.repeat_interleave(2)
        item_tensor = torch.stack((pos_items, neg_items)).t().contiguous().view(-1)
        out = self.forward()
        score = torch.sum(out[user_tensor] * out[item_tensor], dim=1).view(-1, 2)
        loss = -torch.mean(torch.log(torch.sigmoid(torch.matmul(score, self.weight))))
        reg = (self.id_embedding[user_tensor] ** 2 + self.id_embedding[item_tensor] ** 2).mean()
        if self.v_feat is not None:
            reg = reg + (self.v_gcn.preference ** 2).mean()
        return loss + self.reg_weight * reg

    def _score_embeddings(self):
        res = self.result.detach()
        return res[:self.n_users].contiguous(), res[self.n_users:].contiguous()

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
