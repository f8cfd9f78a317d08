"""BPR (matrix factorisation trained with the pairwise BPR loss) on the H100 hot path.  Same class name, constructor,
config keys, parameter names, registration order and `state_dict` order as `src/models/bpr.py`, and the same
construction order (two `nn.Embedding` draws, then `apply(xavier_normal_initialization)`), so `init_seed` gives the
reference's initial weights, and its RNG state after construction, bit for bit.

Kernels:
- Training (`calculate_loss`, `:67-87`): `ops.bpr_mf_loss` on the two embedding tables, with no projected part: the
  gathers, the two row dots, `BPRLoss`, `EmbLoss` and their autograd as one kernel each way; the table gradients are
  scattered by `index_sum_rows`.  `forward`'s `F.dropout(·, 0.0)` returns its input and draws nothing, so the loss does
  not call it.
- Inference (`full_sort_predict`, `:89-95`): `ops.score` of the user rows against the item table; `full_sort_topk`
  inherited."""
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..common.abstract_recommender import GeneralRecommender
from ..common.init import xavier_normal_initialization
from ..common.loss import BPRLoss, EmbLoss


class BPR(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.embedding_size = config["embedding_size"]
        self.reg_weight = config["reg_weight"]
        self.user_embedding = nn.Embedding(self.n_users, self.embedding_size)
        self.item_embedding = nn.Embedding(self.n_items, self.embedding_size)
        self.loss = BPRLoss()
        self.reg_loss = EmbLoss()
        self.apply(xavier_normal_initialization)

    def get_user_embedding(self, user):
        return self.user_embedding(user)

    def get_item_embedding(self, item):
        return self.item_embedding(item)

    def forward(self, dropout=0.0):
        return F.dropout(self.user_embedding.weight, dropout), F.dropout(self.item_embedding.weight, dropout)

    def calculate_loss(self, interaction):
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        return ops.bpr_mf_loss(self.user_embedding.weight, self.item_embedding.weight, None, users, pos_items, neg_items,
                               self.reg_weight)

    def _score_embeddings(self):
        return self._cached_eval_embeddings(lambda: (self.user_embedding.weight, self.item_embedding.weight))

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
