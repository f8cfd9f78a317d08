"""SelfCF's graph encoder on the H100 hot path; mirrors `src/common/encoders.py` (module path, class name `LightGCN_Encoder`,
config keys, `embedding_dict` parameter names and registration order: `init_seed` gives the reference's initial weights
bit for bit and a reference `state_dict` loads with `strict=True`).

`forward` (`:90-112`) draws a fresh edge dropout of the whole normalised adjacency per training batch and propagates
through the dropped matrix.  The reference builds a new un-coalesced sparse tensor from the kept entries and runs
`torch.sparse.mm` on it, forward and backward.  Here the adjacency is the fixed CSR of `graph.build_norm_adj` with its
fixed SpMM plan: the draws are turned into one keep bit per CSR position (`ops.edge_keep_bits`, through the reference's
entry order, `graph.dropout_entry_maps`) and K1 skips the dropped entries (`ops.propagate_mean_dropped`).  No sort, no
rebuilt plan and no host sync per step.

The draws are the reference's, in its order: `np.random.random()` for the rate, then `torch.rand(nnz)` on torch's CPU
generator, copied to the device (`:78-81`).  The keep test `floor(float32(1 - rate) + r)` is one fp32 add and the kept
values are multiplied by `float32(1 / (1 - rate))` in fp32, as torch does both.  `get_embedding` (`:114-131`) propagates the
undropped matrix through the fused inference route."""
import numpy as np
import torch
import torch.nn as nn

from .. import graph, ops
from .abstract_recommender import GeneralRecommender


class LightGCN_Encoder(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.user_count = self.n_users
        self.item_count = self.n_items
        self.latent_size = config["embedding_size"]
        self.n_layers = 3 if config["n_layers"] is None else config["n_layers"]
        self.layers = [self.latent_size] * self.n_layers
        self.drop_ratio = 1.0
        self.drop_flag = True
        self.embedding_dict = self._init_model()
        inter = self.interaction_matrix
        self.sparse_norm_adj = graph.build_norm_adj(inter, self.n_users, self.n_items, self.device)
        draw_of, mirror = graph.dropout_entry_maps(inter.row, inter.col, self.n_users, self.n_items)
        self.draw_of = torch.from_numpy(draw_of).to(self.device)
        self.mirror = torch.from_numpy(mirror).to(self.device)

    def _init_model(self):
        initializer = nn.init.xavier_uniform_
        return nn.ParameterDict({
            "user_emb": nn.Parameter(initializer(torch.empty(self.user_count, self.latent_size))),
            "item_emb": nn.Parameter(initializer(torch.empty(self.item_count, self.latent_size)))})

    def draw_dropout(self):
        """One `sparse_dropout` draw (`encoders.py:77-88`, `:91-93`): (keep bits, mirrored keep bits, scale)."""
        rate = np.random.random() * self.drop_ratio
        draws = torch.rand(self.sparse_norm_adj.nnz).to(self.device)
        keep, keep_t = ops.edge_keep_bits(draws, float(np.float32(1 - rate)), self.draw_of, self.mirror)
        return keep, keep_t, float(np.float32(1. / (1 - rate)))

    def forward(self, inputs):
        ego = torch.cat([self.embedding_dict["user_emb"], self.embedding_dict["item_emb"]], 0)
        if self.drop_flag:
            keep, keep_t, scale = self.draw_dropout()
            all_embeddings = ops.propagate_mean_dropped(self.sparse_norm_adj, ego, len(self.layers), keep, keep_t, scale)
        else:
            all_embeddings = ops.propagate_mean(self.sparse_norm_adj, ego, len(self.layers))
        user_all_embeddings = all_embeddings[:self.user_count, :]
        item_all_embeddings = all_embeddings[self.user_count:, :]
        users, items = inputs[0], inputs[1]
        return user_all_embeddings[users, :], item_all_embeddings[items, :]

    @torch.no_grad()
    def get_embedding(self):
        all_embeddings = ops.propagate_mean_fused(self.sparse_norm_adj, (self.embedding_dict["user_emb"], self.embedding_dict["item_emb"]),
                                                  len(self.layers), cooperative=False)
        return all_embeddings[:self.user_count, :], all_embeddings[self.user_count:, :]
