"""SELFCFED_LGN (SelfCF with embedding dropout) on the H100 hot path; mirrors `src/models/selfcfed_lgn.py` (class name,
config keys, parameter names and registration order: `online_encoder`, then `predictor`).

The encoder is `common.encoders.LightGCN_Encoder`: its per-batch edge dropout runs inside the SpMM (K1 with an edge-keep
mask) instead of a rebuilt sparse matrix.  The predictor, the target dropouts (on the device generator, users first), the
negative-cosine losses and the L2 term are the reference's torch calls in its order.

Scoring (`:71-78`): `P(u)[user] @ i^T + u[user] @ P(i)^T` is ONE product of width 2d, `[P(u) | u] @ [i | P(i)]^T`
(`ops.score`; `full_sort_topk` runs K3's fused score + top-k on the same operands).  The concatenation sums the 2d products
in one fp32 chain instead of two d-chains and an add, so the scores differ from the reference's in the last bits (fp32
reorder error); rankings differ only at near ties."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops
from ..common.abstract_recommender import GeneralRecommender
from ..common.encoders import LightGCN_Encoder
from ..common.loss import L2Loss


class SELFCFED_LGN(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.user_count = self.n_users
        self.item_count = self.n_items
        self.latent_size = config["embedding_size"]
        self.dropout = config["dropout"]
        self.reg_weight = config["reg_weight"]
        self.online_encoder = LightGCN_Encoder(config, dataset)
        self.predictor = nn.Linear(self.latent_size, self.latent_size)
        self.reg_loss = L2Loss()

    def forward(self, inputs):
        u_online, i_online = self.online_encoder(inputs)
        with torch.no_grad():
            u_target, i_target = u_online.clone(), i_online.clone()
            u_target = F.dropout(u_target, self.dropout)
            i_target = F.dropout(i_target, self.dropout)
        return u_online, u_target, i_online, i_target

    @torch.no_grad()
    def get_embedding(self):
        u_online, i_online = self.online_encoder.get_embedding()
        return self.predictor(u_online), u_online, self.predictor(i_online), i_online

    def loss_fn(self, p, z):  # negative cosine similarity
        return - F.cosine_similarity(p, z.detach(), dim=-1).mean()

    def calculate_loss(self, interaction):
        u_online, u_target, i_online, i_target = self.forward(interaction)
        reg_loss = self.reg_loss(u_online, i_online)
        u_online, i_online = self.predictor(u_online), self.predictor(i_online)
        loss_ui = self.loss_fn(u_online, i_target) / 2
        loss_iu = self.loss_fn(i_online, u_target) / 2
        return loss_ui + loss_iu + self.reg_weight * reg_loss

    def _score_embeddings(self):
        """([P(u) | u], [i | P(i)]): the two score products of `full_sort_predict` as one contraction of width 2d."""
        def run():
            pu, u, pi, i = self.get_embedding()
            return torch.cat((pu, u), dim=1), torch.cat((i, pi), dim=1)
        return self._cached_eval_embeddings(run)

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
