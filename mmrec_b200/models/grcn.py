"""GRCN (ACM MM'20) on the H100 hot path; mirrors `src/models/grcn.py` (classes `GRCN`, `EGCN`, `CGCN`, the constructor,
config keys, parameter names `id_gcn.id_embedding`, `v_gcn.preference`, `v_gcn.MLP.*`, `t_gcn.*`, `model_specific_conf`
and their registration order, and the torch draws of the initialisation: `init_seed` gives the reference's initial
`state_dict` and RNG state bit for bit) WITHOUT torch_geometric.

Graph: one CSR over N = U + I nodes (`graph.build_grcn_adj`) holds the reference's symmetric edge list
`cat(edge_index, edge_index[[1, 0]])` (`:158-159`, `:95`), row = target, column = source, every interaction its own entry;
`self.edge_order[e]` is the reference's position of CSR entry e.  `dropout_adj(p=0)` (`:228`) returns its input.

Forward:
- `CGCN` (`:139-166`): `MLP(features)` is `ops.project` (K2; weight and bias gradients by K5's `linear_wgrad`) over the
  frozen feature table, then the reference's `leaky_relu` and `F.normalize`.  The routing loop (`:149-156`) runs GATConv on
  the one-directional list, whose targets `edge_index[1]` are item rows only, so `x_hat_1[:num_user]` is exactly zero
  and carries no gradient: the loop is `preference = F.normalize(preference)` num_routing times, with no graph work (the
  values differ at most in the sign of a zero; tests/test_grcn_host.py).  The one real convolution (`:158-166`) is
  `ops.edge_attention` on `cat(preference, features)` with the base `x`: the scores, PyG's grouped softmax and
  `x + sum alpha x_j` in one row kernel, and alpha in CSR order.
- The edge weights (`:272-281`, `weight_mode = 'confid'`, `pruning`): each modality's alpha times `model_specific_conf` of
  the edge's source node (the `cat` on `:273` takes users' rows for the forward edges, then items' rows), the max over
  modalities, `relu`; torch element-wise ops on [2E, n_modal].
- `EGCN` (`:93-109`): `x = normalize(id_embedding)`, then `x + A_w x + A_w (A_w x)` as two `ops.spmm_values` on the CSR
  with the weights as values, differentiable w.r.t. the weights and x.
- The representation is `cat(id_rep, v_rep[, t_rep])`: 192 wide with both modalities, 128 with the image only.

Evaluation: `full_sort_predict` / `full_sort_topk` score the stored `result` on the exact fp32 route (`ops.score` +
`ops.mask_topk`): the tensor-core scoring stops at d = 128.

Reference quirks kept on purpose:
- `result` is a random [N, embedding_size] table at construction (`:214`), drawn with `torch.rand` + `xavier_normal_`;
  `full_sort_predict` scores the `result` of the last forward (`:296`, `:335-341`): before any training that random table,
  afterwards the representation of the last training batch, taken before its optimizer step.
- Every `nn.init.xavier_normal_(torch.rand(...))` consumes two draws; `MLP` is default-initialised, then `xavier_normal_`
  is applied to its weight (`:134-136`).
- The loss is `-mean(log(sigmoid(.)))`, not `logsigmoid` (`:313`).  The regulariser holds the image preference twice:
  over all users through `reg_embedding_loss +=` (`:316`) and over the batch's users in `reg_content_loss` (`:320`);
  `reg_confid_loss` is computed in the reference but unused (`:326`), so it is not computed here; the loss has shape
  [1], from `torch.zeros(1)` (`:318`).
- `features` is a plain tensor in the reference (not in the `state_dict`); here it is a non-persistent buffer.
- `EGCN.conv_embed_*` and `CGCN.conv_embed_1` hold no parameters; they are not modules here.

Refused at construction with `MMRecError`: text features without image features (the reference's typo `conetent_rep`
(`:257`) leaves `content_rep` None and `torch.cat` fails in the first forward) and no modality at all."""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import graph, ops
from .._lib import MMRecError
from ..common.abstract_recommender import GeneralRecommender


class EGCN(nn.Module):
    """`grcn.py:80-109` with `aggr_mode = 'add'`: both SAGEConvs are products with the weighted symmetric adjacency."""

    def __init__(self, num_user, num_item, dim_E, aggr_mode, has_act, has_norm):
        super().__init__()
        self.num_user, self.num_item, self.dim_E = num_user, num_item, dim_E
        self.aggr_mode, self.has_act, self.has_norm = aggr_mode, has_act, has_norm
        self.id_embedding = nn.Parameter(nn.init.xavier_normal_(torch.rand((num_user + num_item, dim_E))))

    def forward(self, adj: ops.CSR, weight: torch.Tensor):
        x = F.normalize(self.id_embedding) if self.has_norm else self.id_embedding
        x_hat_1 = ops.spmm_values(adj, weight, x)
        if self.has_act:
            x_hat_1 = F.leaky_relu(x_hat_1)
        x_hat_2 = ops.spmm_values(adj, weight, x_hat_1)
        if self.has_act:
            x_hat_2 = F.leaky_relu(x_hat_2)
        return x + x_hat_1 + x_hat_2


class CGCN(nn.Module):
    """`grcn.py:112-166` for a feature table (`is_word = False`, the only form GRCN builds)."""

    def __init__(self, features, num_user, num_item, dim_C, aggr_mode, num_routing, has_act, has_norm, is_word=False):
        super().__init__()
        if is_word:
            raise MMRecError("GRCN: CGCN's word-embedding form (is_word) is not supported; GRCN builds it with is_word = False")
        self.num_user, self.num_item, self.aggr_mode, self.num_routing = num_user, num_item, aggr_mode, num_routing
        self.has_act, self.has_norm, self.dim_C, self.is_word = has_act, has_norm, dim_C, is_word
        self.preference = nn.Parameter(nn.init.xavier_normal_(torch.rand((num_user, dim_C))))
        self.dim_feat = features.size(1)
        self.register_buffer("features", features, persistent=False)
        self.MLP = nn.Linear(self.dim_feat, self.dim_C)
        nn.init.xavier_normal_(self.MLP.weight)

    def forward(self, adj: ops.CSR):
        features = F.leaky_relu(ops.project(self.features, self.MLP.weight, self.MLP.bias))
        preference = self.preference
        if self.has_norm:
            preference = F.normalize(preference)
            features = F.normalize(features)
        for _ in range(self.num_routing):          # x_hat_1[:num_user] == 0: only the normalisation acts (module docstring)
            if self.has_norm:
                preference = F.normalize(preference)
        x = torch.cat((preference, features), dim=0)
        if self.has_act:
            y, alpha = ops.edge_attention(adj, x)
            return x + F.leaky_relu(y), alpha.view(-1, 1)
        y, alpha = ops.edge_attention(adj, x, base=x)
        return y, alpha.view(-1, 1)


class GRCN(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        if self.v_feat is None:
            raise MMRecError("GRCN: no image features.  Text-only fails in the reference (src/models/grcn.py:257: the typo "
                             "`conetent_rep` leaves content_rep None and torch.cat fails) and a model without modality has no "
                             "edge weights; provide image features (with or without text)")
        self.num_user = self.n_users
        self.num_item = self.n_items
        num_user, num_item = self.n_users, self.n_items
        dim_x = config["embedding_size"]
        dim_C = config["latent_embedding"]
        num_layer = config["n_layers"]
        self.aggr_mode = "add"
        self.weight_mode = "confid"
        self.fusion_mode = "concat"
        has_act, has_norm = False, True
        self.weight = torch.tensor([[1.0], [-1.0]]).to(self.device)
        self.reg_weight = config["reg_weight"]
        self.dropout = 0
        train_interactions = dataset.inter_matrix(form="coo").astype(np.float32)
        edge_index = torch.tensor(np.column_stack((train_interactions.row, train_interactions.col + self.n_users)), dtype=torch.long)
        self.edge_index = edge_index.t().contiguous().to(self.device)
        self.attn_adj, self.edge_order = graph.build_grcn_adj(train_interactions, num_user, num_item, self.device)
        self.num_modal = 0
        self.id_gcn = EGCN(num_user, num_item, dim_x, self.aggr_mode, has_act, has_norm)
        self.pruning = True
        num_model = 0
        if self.v_feat is not None:
            self.v_gcn = CGCN(self.v_feat, num_user, num_item, dim_C, self.aggr_mode, num_layer, has_act, has_norm)
            num_model += 1
        if self.t_feat is not None:
            self.t_gcn = CGCN(self.t_feat, num_user, num_item, dim_C, self.aggr_mode, num_layer, has_act, has_norm)
            num_model += 1
        self.model_specific_conf = nn.Parameter(nn.init.xavier_normal_(torch.rand((num_user + num_item, num_model))))
        self.result = nn.init.xavier_normal_(torch.rand((num_user + num_item, dim_x))).to(self.device)

    def edge_weight(self, alphas):
        """`grcn.py:272-281`: [nnz] in CSR order from the modalities' alpha columns [nnz, 1] (image first)."""
        weight = torch.cat(alphas, dim=1)
        src = self.attn_adj.colidx[:self.attn_adj.nnz].to(torch.int64)   # the edge's source node
        weight = weight * self.model_specific_conf[src]
        weight, _ = torch.max(weight, dim=1)
        return torch.relu(weight)

    def forward(self):
        v_rep, weight_v = self.v_gcn(self.attn_adj)
        reps, alphas = [v_rep], [weight_v]
        if self.t_feat is not None:
            t_rep, weight_t = self.t_gcn(self.attn_adj)
            reps.append(t_rep)
            alphas.append(weight_t)
        weight = self.edge_weight(alphas)
        id_rep = self.id_gcn(self.attn_adj, weight)
        representation = torch.cat([id_rep] + reps, dim=1)
        self.result = representation
        return representation

    def calculate_loss(self, interaction):
        batch_users = interaction[0]
        pos_items = interaction[1] + self.n_users
        neg_items = interaction[2] + self.n_users
        user_tensor = batch_users.repeat_interleave(2)
        item_tensor = torch.stack((pos_items, neg_items)).t().contiguous().view(-1)
        out = self.forward()
        score = torch.sum(out[user_tensor] * out[item_tensor], dim=1).view(-1, 2)
        loss = -torch.mean(torch.log(torch.sigmoid(torch.matmul(score, self.weight))))
        reg_embedding_loss = (self.id_gcn.id_embedding[user_tensor] ** 2 + self.id_gcn.id_embedding[item_tensor] ** 2).mean()
        reg_embedding_loss = reg_embedding_loss + (self.v_gcn.preference ** 2).mean()
        reg_content_loss = torch.zeros(1, device=out.device)
        reg_content_loss = reg_content_loss + (self.v_gcn.preference[user_tensor] ** 2).mean()
        if self.t_feat is not None:
            reg_content_loss = reg_content_loss + (self.t_gcn.preference[user_tensor] ** 2).mean()
        reg_loss = self.reg_weight * (reg_embedding_loss + reg_content_loss)
        return loss + reg_loss

    def _score_embeddings(self):
        res = self.result.detach()
        return res[:self.n_users].contiguous(), res[self.n_users:].contiguous()

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])

    def full_sort_topk(self, interaction, k):
        scores = self.full_sort_predict(interaction)
        _, idx = ops.mask_topk(scores, interaction[1], k)
        return idx
