"""VBPR (visual BPR: an item's embedding is its ID row next to a linear projection of its raw features) on the H100 hot
path.  Same class name, constructor, config keys, parameter names, registration order and `state_dict` order as
`src/models/vbpr.py`, and the same construction order (`xavier_uniform_` of `u_embedding` and `i_embedding`,
`nn.Linear`'s default initialisation, then `apply(xavier_normal_initialization)`), so `init_seed` gives the reference's
initial weights, and its RNG state after construction, bit for bit.  `item_raw_features` is the reference's plain
attribute: `cat(t_feat, v_feat)`, text first, or whichever modality exists alone.

Kernels:
- Training (`calculate_loss`, `:77-98`): the reference projects the whole raw table (`forward`, `:69-75`) and reads 2B
  of its rows.  The projection is row-wise and the table is frozen, so the model projects only `cat(pos, neg)` (K2
  with `idx`; its backward is K5's weight and bias gradients over the same rows), which gives the rows the loss reads
  and the weight and bias gradients of the full-table route.  `ops.bpr_mf_loss` then reads `[i_embedding[item] |
  projected row]` itself (no concatenated table) and runs the gathers, dots, `BPRLoss`, `EmbLoss` and their autograd as
  one kernel each way.  `F.dropout(·, 0.0)` returns its input and draws nothing, so the loss does not call it.
- Inference (`full_sort_predict`, `:100-106`, under the evaluation cache): `(u_embedding, cat(i_embedding, K2 over all
  items))`, 128 wide, and `ops.score`; `full_sort_topk` inherited.

Departure from the reference: `get_item_embedding` (`:58-67`) reads `self.item_embedding`, which VBPR never defines, so
it cannot run there; it is left out."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..common.abstract_recommender import GeneralRecommender
from ..common.init import xavier_normal_initialization
from ..common.loss import BPRLoss, EmbLoss


class VBPR(GeneralRecommender):
    def __init__(self, config, dataloader):
        super().__init__(config, dataloader)
        self.u_embedding_size = self.i_embedding_size = config["embedding_size"]
        self.reg_weight = config["reg_weight"]
        self.u_embedding = nn.Parameter(nn.init.xavier_uniform_(torch.empty(self.n_users, self.u_embedding_size * 2)))
        self.i_embedding = nn.Parameter(nn.init.xavier_uniform_(torch.empty(self.n_items, self.i_embedding_size)))
        if self.v_feat is not None and self.t_feat is not None:
            self.item_raw_features = torch.cat((self.t_feat, self.v_feat), -1)
        elif self.v_feat is not None:
            self.item_raw_features = self.v_feat
        else:
            self.item_raw_features = self.t_feat
        self.item_linear = nn.Linear(self.item_raw_features.shape[1], self.i_embedding_size)
        self.loss = BPRLoss()
        self.reg_loss = EmbLoss()
        self.apply(xavier_normal_initialization)

    def get_user_embedding(self, user):
        return self.u_embedding[user, :]

    def forward(self, dropout=0.0):
        item_embeddings = ops.project(self.item_raw_features, self.item_linear.weight, self.item_linear.bias)
        item_embeddings = torch.cat((self.i_embedding, item_embeddings), -1)
        return F.dropout(self.u_embedding, dropout), F.dropout(item_embeddings, dropout)

    def calculate_loss(self, interaction):
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        both = torch.cat((pos_items, neg_items))
        proj = ops.project(self.item_raw_features, self.item_linear.weight, self.item_linear.bias, idx=both)   # only these rows
        return ops.bpr_mf_loss(self.u_embedding, self.i_embedding, proj, users, pos_items, neg_items, self.reg_weight)

    def _score_embeddings(self):
        return self._cached_eval_embeddings(lambda: self.forward())

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
