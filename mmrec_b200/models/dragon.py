"""DRAGON (arXiv'23) on the H100 hot path; mirrors `src/models/dragon.py` (class `DRAGON`, the constructor, config keys,
parameter names, registration order and the torch and `np.random` consumption of the initialisation: `init_seed` gives the
reference's initial weights bit for bit and a reference `state_dict` from the GPU loads with `strict=True`) WITHOUT
torch_geometric.  Its `GCN`, `Base_gcn`, `User_Graph_sample` and `topk_sample` are DualGNN's (`dragon.py:287-416` =
`dualgnn.py:207-345`), so they are `dualgnn`'s classes here; its item graph `mm_adj` is FREEDOM's (`dragon.py:61-83,
158-179` = `freedom.py:67-100`), `graph.build_freedom_mm_adj`.

Kernels:
- Both modality towers' convs are one propagation, as in DualGNN: `ops.propagate_sum` at L = 2 on [x_v | x_t] with the
  'add' (`graph.build_gcn_add_adj`) or 'mean' (`mmgcn.mean_adj_from_edges`) adjacency.  With `construction = 'cat'`
  (`:44`) its [N, 128] output IS `representation` (`:206`): nothing is concatenated.
- `user_rep` is the reference's torch weighting and `cat`s (`:237-243`).  The user graph `user_rep + h_u1` (`:251-252`)
  is `ops.spmm` on the epoch's user graph G (`graph.build_user_graph`) with `user_rep` as the epilogue's base: no U x 40 x
  d gather.  The item graph `item_rep + mm_adj^n_mm_layers item_rep` (`:248-253`) is `ops.spmm` per product, the last
  one adding `item_rep` in its epilogue; its backward reads mm_adj's transpose, built once at construction.  A weighting
  kernel with both graph products in one SpMM launch measured no faster than this on an H100 (DESIGN.md, n10), so the
  model does not use one.
- `MLP(features)` is `ops.project` at width 256 with its bias (K2 forward, `linear_wgrad` backward).
- Scoring is `ops.score` / `ops.score_topk` on `result_embed` through `_score_embeddings` and the evaluation cache.

Reference quirks kept on purpose:
- `pos_item_nodes += self.n_users` and `neg_item_nodes += self.n_users` mutate the caller's batch tensors (`:193-194`).
- `v_preference` and `t_preference` are None until the first forward assigns the towers' preferences to them (`:198,
  201`); from then on they are registered attributes of the model.
- `weight_i`, `MLP_v`, `MLP_t`, `MLP_user`, `image_embedding`, `text_embedding`, `image_trs` and `text_trs` are
  registered but get no gradient: nothing in the loss reads them (`:53-54`, `:64-68`, `:96-98`, `:140`).
- `n_layers` is unused: `num_layer = 1` (`:40`), and the one conv is applied twice, `x_hat = h + x + h_1` (`:379-382`).
- `full_sort_predict` scores the `result_embed` of the last forward (`:254`, `:279-285`): the last training batch's
  forward, taken before its optimizer step.
- Before any forward, `result_embed` is the initial float64 [U + I, embedding_size] tensor (`:155-156`), so the scores
  are float64; that path stays a torch matmul on the device, and `full_sort_topk` masks and ranks those float64 scores as
  the trainer does.  After a forward it is float32 and 128 wide (64 with one modality).
- `result_embed` is never a parameter: the reference's `nn.Parameter(...).to(device)` returns a plain tensor on the GPU.
- The loss is `-mean(log2(sigmoid(pos - neg)))` plus `reg_weight` times the users' preference means and the mean of
  `weight_u ** 2` (`:262-277`, the 'cat' branch).
- The dropped-item edge lists `edge_index_dropv` / `edge_index_dropt` and `v_drop_ze` / `t_drop_ze` (`:100-151`) are
  never read (`GCN.forward` ignores `edge_index_drop`).  The `np.random.choice` behind them is drawn, so the RNG stream
  stays the reference's; the lists themselves are not built.
Departures:
- `mm_adj` is built in memory at construction, from the feature tables, and the model neither reads nor writes
  `mm_adj_{knn_k}.pt`.  The reference loads that file when it exists, without checking that it belongs to the same
  features, `knn_k` or `mm_image_weight` (`:61-83`), and writes it otherwise.
- `aggr_mode` must be 'add' or 'mean'; anything else raises `MMRecError` at construction, where the reference fails on
  the first forward.
Supported: either modality alone, as the reference's `forward` allows: then there is no weighting and the width is 64."""
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from .._lib import MMRecError
from ..common.abstract_recommender import GeneralRecommender
from .dualgnn import GCN, User_Graph_sample
from .mmgcn import mean_adj_from_edges

AGGR_MODES = ("add", "mean")


class DRAGON(GeneralRecommender):
    _eval_cache_deps = GeneralRecommender._eval_cache_deps + ("result_embed",)

    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        num_user = self.n_users
        num_item = self.n_items
        batch_size = config["train_batch_size"]
        dim_x = config["embedding_size"]
        self.feat_embed_dim = config["feat_embed_dim"]
        self.n_layers = config["n_mm_layers"]
        self.knn_k = config["knn_k"]
        self.mm_image_weight = config["mm_image_weight"]
        has_id = True
        self.batch_size = batch_size
        self.num_user = num_user
        self.num_item = num_item
        self.k = 40
        self.aggr_mode = config["aggr_mode"]
        if self.aggr_mode not in AGGR_MODES:
            raise MMRecError(f"DRAGON: aggr_mode {self.aggr_mode!r} is not supported (one of {AGGR_MODES})")
        self.user_aggr_mode = "softmax"
        self.num_layer = 1
        self.cold_start = 0
        self.dataset = dataset
        self.construction = "cat"
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

        if self.v_feat is not None:
            self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=False)
            self.image_trs = nn.Linear(self.v_feat.shape[1], self.feat_embed_dim)
        if self.t_feat is not None:
            self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=False)
            self.text_trs = nn.Linear(self.t_feat.shape[1], self.feat_embed_dim)
        # w * image_adj + (1 - w) * text_adj, built here every time (no mm_adj_{k}.pt, module docstring); its transpose
        # is the backward's
        self.mm_adj = graph.build_freedom_mm_adj(self.v_feat, self.t_feat, self.knn_k, self.mm_image_weight)
        self.mm_adj.t()

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
        # the draw behind the unused dropped-item edge lists (dragon.py:100-138): consumed, the lists are not built
        drop_item = torch.tensor(np.random.choice(self.item_index.numpy(), int(self.num_item * self.drop_percent), replace=False))
        drop_item_single = drop_item[:int(self.single_percent * len(drop_item))]
        self.dropv_node_idx_single = drop_item_single[:int(len(drop_item_single) * 1 / 3)]
        self.dropt_node_idx_single = drop_item_single[int(len(drop_item_single) * 2 / 3):]
        self.dropv_node_idx = self.dropv_node_idx_single
        self.dropt_node_idx = self.dropt_node_idx_single

        self.MLP_user = nn.Linear(self.dim_latent * 2, self.dim_latent)
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
        """`topk_sample(k)` (`:181-183`) on the host, then the epoch's user graph as a device CSR and its transpose."""
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
            raise MMRecError("DRAGON: no user graph yet: pre_epoch_processing() samples it before each epoch")
        towers = [g for g in (getattr(self, "v_gcn", None), getattr(self, "t_gcn", None)) if g is not None]
        feats = [f for f in (self.v_feat, self.t_feat) if f is not None]
        x = torch.cat([g.embed(f) for g, f in zip(towers, feats)], dim=1) if len(towers) > 1 else towers[0].embed(feats[0])
        out = ops.propagate_sum(self.adj, x, 2)                        # [v_rep | t_rep] = the 'cat' representation
        d = self.dim_latent
        if self.v_feat is not None:
            self.v_rep, self.v_preference = out[:, :d], self.v_gcn.preference
        if self.t_feat is not None:
            self.t_rep, self.t_preference = out[:, -d:], self.t_gcn.preference
        if self.v_feat is not None and self.t_feat is not None:
            self.v_rep, self.t_rep = torch.unsqueeze(self.v_rep, 2), torch.unsqueeze(self.t_rep, 2)
            user_rep = torch.cat((self.v_rep[:self.num_user], self.t_rep[:self.num_user]), dim=2)
            user_rep = self.weight_u.transpose(1, 2) * user_rep
            user_rep = torch.cat((user_rep[:, :, 0], user_rep[:, :, 1]), dim=1)
        else:
            user_rep = out[:self.num_user]
        item_rep = out[self.num_user:]
        h = item_rep
        for _ in range(self.n_layers - 1):
            h = ops.spmm(self.mm_adj, h)
        item_rep = ops.spmm(self.mm_adj, h, base=item_rep) if self.n_layers > 0 else item_rep + h   # item_rep + h, fused
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
        return loss_value + reg_loss

    def _score_embeddings(self):
        res = self.result_embed.detach()
        return self._cached_eval_embeddings(lambda: (res[:self.n_users].contiguous(), res[self.n_users:].contiguous()))

    def _initial_scores(self, users):
        """Before any forward: the float64 product of the initial `result_embed` (`:279-285`), a torch matmul on the device."""
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
