"""ItemKNNCBF on the H100 hot path; mirrors `src/models/itemknncbf.py` (class name, config keys `knn_k` / `shrink`, the
`dummy_embeddings` parameter, features `cat(v_feat, t_feat)` or the one modality present).

The reference builds a dense [I, I] similarity graph (`build_item_sim_matrix`, `:56-65`) and keeps the dense [U, I]
product `scores_matrix = torch.mm(R, item_sim)` (`:54`) for the life of the model: 2.1 GB + 3.7 GB at clothing's shape,
62.5 GB for the graph alone at 125 037 items.  This class holds neither.  Both are sparse in what they keep:

* the graph has `knn_k` entries per row: K7's shrink route (`ops.knn_topk(.., norms=, shrink=)`) ranks
  `(X X^T) / (|x_i||x_j| + shrink)` without the [I, I] matrix, and the result is kept as a CSR `item_sim`;
* a user's score row has at most deg(u) * knn_k non-zeros: K9 (`ops.sparse_scores`, `ops.sparse_score_topk`) forms it
  from the interaction CSR `r_matrix` and `item_sim` per evaluation batch, summing over R's row in ascending column order.
"""
import numpy as np
import torch
import torch.nn as nn

from .. import ops
from ..common.abstract_recommender import GeneralRecommender


class ItemKNNCBF(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.knn_k = config["knn_k"]
        self.shrink = config["shrink"]

        inter = dataset.inter_matrix(form="coo").astype(np.float32)
        self.r_matrix = ops.CSR.from_coo(torch.from_numpy(inter.row.astype(np.int64)).to(self.device),
                                         torch.from_numpy(inter.col.astype(np.int64)).to(self.device),
                                         torch.from_numpy(inter.data.astype(np.float32)).to(self.device), self.n_users, self.n_items)

        if self.v_feat is not None and self.t_feat is not None:
            item_fea = torch.cat((self.v_feat, self.t_feat), -1)
        elif self.v_feat is not None:
            item_fea = self.v_feat
        else:
            item_fea = self.t_feat

        self.dummy_embeddings = nn.Parameter(torch.Tensor([0.5, 0.5]))

        self.item_sim = self.build_item_sim_matrix(item_fea)

    def build_item_sim_matrix(self, features):
        """The `knn_k` largest `sim[i, :]` per item, `sim = (X X^T) / (i_norm i_norm^T + shrink)`, as a CSR [I, I]
        (the reference's scatter into a dense matrix, `:56-65`).  The norms are the reference's expression."""
        n = features.shape[0]
        i_norm = torch.norm(features, p=2, dim=-1)
        val, idx = ops.knn_topk(features, self.knn_k, norms=i_norm, shrink=float(self.shrink))
        rows = torch.arange(n, device=features.device).repeat_interleave(self.knn_k)
        return ops.CSR.from_coo(rows, idx.reshape(-1), val.reshape(-1), n, n)

    def calculate_loss(self, interaction):
        return torch.tensor(0.0)

    def full_sort_predict(self, interaction):
        return ops.sparse_scores(self.r_matrix, self.item_sim, interaction[0])

    def full_sort_topk(self, interaction, k):
        """`full_sort_predict` + `scores[mask] = -1e10` + `torch.topk(scores, k)` (`src/common/trainer.py:304-309`) without
        a dense score row; returns the index matrix only, like the trainer keeps."""
        _, idx = ops.sparse_score_topk(self.r_matrix, self.item_sim, interaction[0], interaction[1], k)
        return idx
