"""DualGNN (TMM'21) on the H100 hot path; mirrors `src/models/dualgnn.py` (classes `DualGNN`, `GCN`, `Base_gcn`,
`User_Graph_sample`, the constructor, config keys, parameter names, registration order and the torch and `np.random`
consumption of the initialisation: `init_seed` gives the reference's initial weights bit for bit and a reference
`state_dict` from the GPU loads with `strict=True`) WITHOUT torch_geometric.

Kernels:
- Both modality towers' convs are one propagation.  `Base_gcn` (`:318-345`) is the SpMM with PyG's gcn norm (`'add'`,
  `graph.build_gcn_add_adj`) or the row-normalised mean adjacency (`'mean'`, `mmgcn.mean_adj_from_edges`).  The tower's
  `h = conv(x)`, `h_1 = conv(h)`, `x_hat = h + x + h_1` (`:311-314`) is `ops.propagate_sum` at L = 2, run once on the
  [N, 128] table `[x_v | x_t]`; the towers are its column blocks.
- `User_Graph_sample` (`:252-266`: a [U, 40, 64] gather of a Python list index, then a batched matmul) is `ops.spmm` on
  the per-epoch user graph G, a CSR built in `pre_epoch_processing`, with `user_rep` as the epilogue's base: no U x 40 x d
  tensor, no list converted per batch.
- `MLP(features)` is `ops.project` at width 256 with its bias (K2 forward, `linear_wgrad` backward); `leaky_relu`, `MLP_1`,
  the concatenation with `preference` and `F.normalize` stay torch, in the reference's order.
- Scoring is `ops.score` / `ops.score_topk` on `result_embed` through `_score_embeddings` and the evaluation cache.

Reference quirks kept on purpose:
- `representation += self.t_rep` is in place (`:154`), so `v_rep` is v + t when the weighted sum reads it:
  user_rep = (v + t) w_0 + t w_1 and item_rep = (v + t)[U:].
- `pos_item_nodes += self.n_users` and `neg_item_nodes += self.n_users` mutate the caller's batch tensors (`:143-144`).
- `weight_i` enters the loss only through the regulariser (`:194`); `MLP_v`, `MLP_t` and `MLP_user` are registered but
  unused (`:49-50`, `:113`).
- `n_layers` is unused: `num_layer = 1` (`:36`), and the one conv is applied twice, `x_hat = h + x + h_1` (`:311-314`).
- `full_sort_predict` scores the `result_embed` of the last forward (`:174`, `:199-205`): the last training batch's
  forward, taken before its optimizer step.
- Before any forward, `result_embed` is the initial float64 tensor (`:129`), so the scores are float64; that path stays
  a torch matmul on the device, and `full_sort_topk` masks and ranks those float64 scores as the trainer does.
- `result_embed` is never a parameter: the reference's `nn.Parameter(...).to(device)` returns a plain tensor on the GPU.
- The loss is `-mean(log2(sigmoid(pos - neg)))` plus `reg_weight` times the users' preference means and the means of
  `weight_u ** 2` and `weight_i ** 2` (`:185-197`).
- The dropped-item edge lists `edge_index_dropv` / `edge_index_dropt` and `v_drop_ze` / `t_drop_ze` (`:92-111`, `:117`,
  `:122`) are built but never read.  The `np.random.choice` behind them is drawn, so the RNG stream stays the
  reference's; the lists themselves are not built.
Supported: `aggr_mode` 'add' and 'mean' (anything else raises `MMRecError`), and either modality alone, as the
reference's `forward` allows."""
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from .._lib import MMRecError
from ..common.abstract_recommender import GeneralRecommender
from .mmgcn import mean_adj_from_edges

AGGR_MODES = ("add", "mean")


class DualGNN(GeneralRecommender):
    _eval_cache_deps = GeneralRecommender._eval_cache_deps + ("result_embed",)

    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        num_user = self.n_users
        num_item = self.n_items
        batch_size = config["train_batch_size"]
        dim_x = config["embedding_size"]
        has_id = True
        self.batch_size = batch_size
        self.num_user = num_user
        self.num_item = num_item
        self.k = 40
        self.aggr_mode = config["aggr_mode"]
        if self.aggr_mode not in AGGR_MODES:
            raise MMRecError(f"DualGNN: aggr_mode {self.aggr_mode!r} is not supported (one of {AGGR_MODES})")
        self.user_aggr_mode = "softmax"
        self.num_layer = 1
        self.cold_start = 0
        self.dataset = dataset
        self.construction = "weighted_sum"
        self.reg_weight = config["reg_weight"]
        self.drop_rate = 0.1
        self.v_rep = None
        self.t_rep = None
        self.v_preference = None
        self.t_preference = None
        self.dim_latent = 64
        self.dim_feat = 128
        self.MLP_v = nn.Linear(self.dim_latent, self.dim_latent, bias=False)
        self.MLP_t = nn.Linear(self.dim_latent, self.dim_latent, bias=False)

        dataset_path = os.path.abspath(config["data_path"] + config["dataset"])
        self.user_graph_dict = np.load(os.path.join(dataset_path, config["user_graph_dict_file"]), allow_pickle=True).item()
        self.user_graph_table = graph.UserGraphTable(self.user_graph_dict, self.k)

        train_interactions = dataset.inter_matrix(form="coo").astype(np.float32)
        edge_index = self.pack_edge_index(train_interactions)
        self.edge_index = torch.tensor(edge_index, dtype=torch.long).t().contiguous().to(self.device)
        self.edge_index = torch.cat((self.edge_index, self.edge_index[[1, 0]]), dim=1)
        n_nodes = num_user + num_item
        if self.aggr_mode == "add":
            self.adj = graph.build_gcn_add_adj(self.edge_index, n_nodes, self.device)
        else:
            self.adj = mean_adj_from_edges(self.edge_index, n_nodes)

        self.weight_u = nn.Parameter(nn.init.xavier_normal_(
            torch.tensor(np.random.randn(self.num_user, 2, 1), dtype=torch.float32, requires_grad=True)))
        self.weight_u.data = F.softmax(self.weight_u.data, dim=1)
        self.weight_i = nn.Parameter(nn.init.xavier_normal_(
            torch.tensor(np.random.randn(self.num_item, 2, 1), dtype=torch.float32, requires_grad=True)))
        self.weight_i.data = F.softmax(self.weight_i.data, dim=1)

        self.item_index = torch.arange(self.num_item, dtype=torch.long)
        self.drop_percent = self.drop_rate
        self.single_percent = 1
        self.double_percent = 0
        # the draw behind the unused dropped-item edge lists (dualgnn.py:80-111): consumed, the lists are not built
        drop_item = torch.tensor(np.random.choice(self.item_index.numpy(), int(self.num_item * self.drop_percent), replace=False))
        drop_item_single = drop_item[:int(self.single_percent * len(drop_item))]
        self.dropv_node_idx_single = drop_item_single[:int(len(drop_item_single) * 1 / 3)]
        self.dropt_node_idx_single = drop_item_single[int(len(drop_item_single) * 2 / 3):]
        self.dropv_node_idx = self.dropv_node_idx_single
        self.dropt_node_idx = self.dropt_node_idx_single

        self.MLP_user = nn.Linear(self.dim_latent * 3, self.dim_latent)
        if self.v_feat is not None:
            self.v_gcn = GCN(self.dataset, batch_size, num_user, num_item, dim_x, self.aggr_mode, num_layer=self.num_layer,
                             has_id=has_id, dropout=self.drop_rate, dim_latent=64, device=self.device, features=self.v_feat)
        if self.t_feat is not None:
            self.t_gcn = GCN(self.dataset, batch_size, num_user, num_item, dim_x, self.aggr_mode, num_layer=self.num_layer,
                             has_id=has_id, dropout=self.drop_rate, dim_latent=64, device=self.device, features=self.t_feat)
        self.user_graph = User_Graph_sample(num_user, "add", self.dim_latent)
        self.result_embed = nn.init.xavier_normal_(torch.tensor(np.random.randn(num_user + num_item, dim_x))).to(self.device)
        self.epoch_user_graph = self.user_weight_matrix = self.user_graph_csr = None

    def pre_epoch_processing(self):
        """`topk_sample(k)` (`:131-133`) on the host, then the epoch's user graph as a device CSR and its transpose."""
        idx, weights = self.topk_sample(self.k)
        self.epoch_user_graph = torch.from_numpy(idx)
        self.user_weight_matrix = torch.from_numpy(weights).to(self.device)
        self.user_graph_csr = graph.build_user_graph(idx, weights, self.device)

    def pack_edge_index(self, inter_mat):
        return np.column_stack((inter_mat.row, inter_mat.col + self.n_users))

    def topk_sample(self, k):
        """(index int64 [U, k], weights fp32 [U, k]) of the reference's `topk_sample` (`graph.UserGraphTable.sample`)."""
        if k != self.user_graph_table.k:
            self.user_graph_table = graph.UserGraphTable(self.user_graph_dict, k)
        return self.user_graph_table.sample(np.random)

    def forward(self, interaction):
        user_nodes, pos_item_nodes, neg_item_nodes = interaction[0], interaction[1], interaction[2]
        pos_item_nodes += self.n_users
        neg_item_nodes += self.n_users
        if self.user_graph_csr is None:
            raise MMRecError("DualGNN: no user graph yet: pre_epoch_processing() samples it before each epoch")
        towers = [g for g in (getattr(self, "v_gcn", None), getattr(self, "t_gcn", None)) if g is not None]
        feats = [f for f in (self.v_feat, self.t_feat) if f is not None]
        x = torch.cat([g.embed(f) for g, f in zip(towers, feats)], dim=1) if len(towers) > 1 else towers[0].embed(feats[0])
        out = ops.propagate_sum(self.adj, x, 2)                        # [x_v | x_t] + h + h_1 for both towers at once
        d = self.dim_latent
        representation = None
        if self.v_feat is not None:
            self.v_rep, self.v_preference = out[:, :d], self.v_gcn.preference
            representation = self.v_rep
        if self.t_feat is not None:
            self.t_rep, self.t_preference = out[:, -d:], self.t_gcn.preference
            if representation is None:
                representation = self.t_rep
            else:
                representation = self.v_rep = self.v_rep + self.t_rep   # sic: the reference's += on v_rep (dualgnn.py:154)
        if self.v_rep is not None:
            self.v_rep = torch.unsqueeze(self.v_rep, 2)
            user_rep = self.v_rep[:self.num_user]
        if self.t_rep is not None:
            self.t_rep = torch.unsqueeze(self.t_rep, 2)
            user_rep = self.t_rep[:self.num_user]
        if self.v_rep is not None and self.t_rep is not None:
            user_rep = torch.matmul(torch.cat((self.v_rep[:self.num_user], self.t_rep[:self.num_user]), dim=2), self.weight_u)
        user_rep = torch.squeeze(user_rep)
        item_rep = representation[self.num_user:]
        user_rep = self.user_graph(user_rep, self.user_graph_csr, self.user_weight_matrix, base=user_rep)   # user_rep + h_u1
        self.result_embed = torch.cat((user_rep, item_rep), dim=0)
        user_tensor = self.result_embed[user_nodes]
        pos_item_tensor = self.result_embed[pos_item_nodes]
        neg_item_tensor = self.result_embed[neg_item_nodes]
        pos_scores = torch.sum(user_tensor * pos_item_tensor, dim=1)
        neg_scores = torch.sum(user_tensor * neg_item_tensor, dim=1)
        return pos_scores, neg_scores

    def calculate_loss(self, interaction):
        user = interaction[0]
        pos_scores, neg_scores = self.forward(interaction)
        loss_value = -torch.mean(torch.log2(torch.sigmoid(pos_scores - neg_scores)))
        reg_embedding_loss_v = (self.v_preference[user] ** 2).mean() if self.v_preference is not None else 0.0
        reg_embedding_loss_t = (self.t_preference[user] ** 2).mean() if self.t_preference is not None else 0.0
        reg_loss = self.reg_weight * (reg_embedding_loss_v + reg_embedding_loss_t)
        reg_loss += self.reg_weight * (self.weight_u ** 2).mean()
        reg_loss += self.reg_weight * (self.weight_i ** 2).mean()
        return loss_value + reg_loss

    def _score_embeddings(self):
        res = self.result_embed.detach()
        return self._cached_eval_embeddings(lambda: (res[:self.n_users].contiguous(), res[self.n_users:].contiguous()))

    def _initial_scores(self, users):
        """Before any forward: the float64 product of the initial `result_embed` (`:199-205`), a torch matmul on the device."""
        res = self.result_embed.detach()
        return torch.matmul(res[:self.n_users][users, :], res[self.n_users:].t())

    def full_sort_predict(self, interaction):
        if self.result_embed.dtype == torch.float64:
            return self._initial_scores(interaction[0])
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])

    def full_sort_topk(self, interaction, k):
        if self.result_embed.dtype == torch.float64:                   # the trainer's mask + top-k of the float64 scores
            scores = self._initial_scores(interaction[0])
            mask = interaction[1]
            scores[mask[0], mask[1]] = -1e10
            return torch.topk(scores, k, dim=-1)[1]
        return super().full_sort_topk(interaction, k)


class User_Graph_sample(nn.Module):
    """`:252-266`: `matmul(weights.unsqueeze(1), features[index]).squeeze()`, as `G @ features` on the epoch's user graph
    (`graph.build_user_graph`); `base` is added in the SpMM's epilogue (`user_rep + h_u1`, `:172-173`)."""

    def __init__(self, num_user, aggr_mode, dim_latent):
        super().__init__()
        self.num_user = num_user
        self.dim_latent = dim_latent
        self.aggr_mode = aggr_mode

    def forward(self, features, user_graph, user_matrix=None, base=None):
        return ops.spmm(user_graph, features, base=base)


class GCN(nn.Module):
    """`:269-315`: one modality tower.  `embed` is its input x; the model propagates the towers together."""

    def __init__(self, datasets, batch_size, num_user, num_item, dim_id, aggr_mode, num_layer, has_id, dropout,
                 dim_latent=None, device=None, features=None):
        super().__init__()
        self.batch_size = batch_size
        self.num_user = num_user
        self.num_item = num_item
        self.datasets = datasets
        self.dim_id = dim_id
        self.dim_feat = features.size(1)
        self.dim_latent = dim_latent
        self.aggr_mode = aggr_mode
        self.num_layer = num_layer
        self.has_id = has_id
        self.dropout = dropout
        self.device = device
        if self.dim_latent:
            self.preference = nn.Parameter(nn.init.xavier_normal_(torch.tensor(
                np.random.randn(num_user, self.dim_latent), dtype=torch.float32, requires_grad=True), gain=1).to(self.device))
            self.MLP = nn.Linear(self.dim_feat, 4 * self.dim_latent)
            self.MLP_1 = nn.Linear(4 * self.dim_latent, self.dim_latent)
            self.conv_embed_1 = Base_gcn(self.dim_latent, self.dim_latent, aggr=self.aggr_mode)
        else:
            self.preference = nn.Parameter(nn.init.xavier_normal_(torch.tensor(
                np.random.randn(num_user, self.dim_feat), dtype=torch.float32, requires_grad=True), gain=1).to(self.device))
            self.conv_embed_1 = Base_gcn(self.dim_latent, self.dim_latent, aggr=self.aggr_mode)

    def embed(self, features):
        """`F.normalize(cat(preference, MLP_1(leaky_relu(MLP(features)))))` (`:306-309`), `MLP` on K2."""
        if self.dim_latent:
            temp_features = self.MLP_1(F.leaky_relu(ops.project(features, self.MLP.weight, self.MLP.bias)))
        else:
            temp_features = features
        x = torch.cat((self.preference, temp_features), dim=0)
        return F.normalize(x)

    def forward(self, adj, features):
        """The tower alone: (x + h + h_1, preference)."""
        return ops.propagate_sum(adj, self.embed(features), 2), self.preference


class Base_gcn(nn.Module):
    """`:318-345`: one propagation step, `adj @ x`, with the 'add' or 'mean' adjacency the model built."""

    def __init__(self, in_channels, out_channels, normalize=True, bias=True, aggr="add", **kwargs):
        super().__init__()
        self.aggr = aggr
        self.in_channels = in_channels
        self.out_channels = out_channels

    def forward(self, x, adj, size=None):
        return ops.spmm(adj, x)
