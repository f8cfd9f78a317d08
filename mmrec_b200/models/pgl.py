"""PGL (principal graph learning: LightGCN on a per-epoch principal sub-graph, plus FREEDOM's frozen item graph and a
self-contrastive InfoNCE on dropout views) on the H100 hot path.  Same class name, constructor, config keys, parameter
names and registration order as `src/models/pgl.py` (`user_text`, `user_image`, `image_embedding`, `image_trs`,
`text_embedding`, `text_trs`), and the same construction order (`nn.Embedding`'s normal draws, `xavier_uniform_` of
`user_image` then `user_text`, `nn.Linear`'s default initialisation, image first), so `init_seed` gives the reference's
initial weights, and its RNG state after construction, bit for bit.

Its shipped configuration, `mode: local`, is built from parts the package already pins:
- `pre_epoch_processing` (`:168-181`): FREEDOM's degree-sensitive pruning (graph.EdgePruner, the same
  `torch.multinomial(edge_values, int(nnz * 0.3))` draw);
- the item graph (`:62-75, 86-107`): FREEDOM's `mm_adj` (graph.build_freedom_mm_adj), built at construction every time:
  the model neither reads nor writes the reference's `mm_adj_freedomdsp_*.pt`;
- `forward` (`:204-225`): K2 with `l2_normalize` for the two projected feature tables, LightGCN's mean (ops.propagate_mean)
  at width 2d on the sub-graph, and `i_g + mm_adj^n @ item_embeds` with the last product's epilogue adding i_g.
  Inference runs `ops.propagate_mean_fused` with the item-item product in layer 1's launch;
- `calculate_loss` (`:244-259`): the four `self.dropoutf` draws, made as the reference makes them (see `_dropout_masks`),
  then `ops.pgl_loss` -- the gathers, BPR, the four views, F.normalize, the positive dots, InfoNCE and their autograd as one
  row kernel each way, with K8 (`ops.expsum_rows`) for the two B x B sums;
- `full_sort_predict` (`:261-269`) on `ops.score`, `full_sort_topk` inherited.

Refused at construction (MMRecError): `mode: global` (the reference's `global_subgraph_extraction` needs `sparsesvd`, which
is not in its own requirements, and forms a dense N x N product), a missing modality (`forward` reads both), and
`feat_embed_dim != embedding_size` (the user and item tables would not concatenate).  `alignment`, `uniformity` and `save`
are never called by the reference and are left out."""
import numpy as np
import torch
import torch.nn as nn

from .. import graph, ops
from .._lib import MMRecError
from ..common.abstract_recommender import GeneralRecommender


class PGL(GeneralRecommender):
    def __init__(self, config, dataset):
        super().__init__(config, dataset)
        self.mode = config["mode"]
        self.embedding_dim = config["embedding_size"]
        self.feat_embed_dim = config["feat_embed_dim"]
        self.knn_k = config["knn_k"]
        self.lambda_coeff = config["lambda_coeff"]
        self.n_layers = config["n_mm_layers"]
        self.n_ui_layers = config["n_ui_layers"]
        self.reg_weight = config["reg_weight"]
        self.mm_image_weight = config["mm_image_weight"]
        if self.mode != "local":
            raise MMRecError(f"PGL: mode {self.mode!r} is not supported: the reference's global sub-graph needs `sparsesvd` "
                             "(not in its requirements) and a dense N x N product; use mode 'local'")
        if self.v_feat is None or self.t_feat is None:
            raise MMRecError("PGL: needs both the image and the text features (the reference's forward reads both)")
        if self.feat_embed_dim != self.embedding_dim:
            raise MMRecError(f"PGL: feat_embed_dim = {self.feat_embed_dim} must equal embedding_size = {self.embedding_dim}: "
                             "the reference concatenates the user and item tables")
        self.n_nodes = self.n_users + self.n_items
        self.sub_graph, self.mm_adj = None, None

        self.interaction_matrix = dataset.inter_matrix(form="coo").astype(np.float32)
        self.norm_adj = graph.build_norm_adj(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.pruner = graph.EdgePruner(self.interaction_matrix, self.n_users, self.n_items, self.device)
        self.edge_indices, self.edge_values = self.pruner.edge_indices, self.pruner.edge_values

        self.user_text = nn.Embedding(self.n_users, self.embedding_dim)
        self.user_image = nn.Embedding(self.n_users, self.embedding_dim)
        nn.init.xavier_uniform_(self.user_image.weight)
        nn.init.xavier_uniform_(self.user_text.weight)
        self.image_embedding = nn.Embedding.from_pretrained(self.v_feat, freeze=False)
        self.image_trs = nn.Linear(self.v_feat.shape[1], self.feat_embed_dim)
        self.text_embedding = nn.Embedding.from_pretrained(self.t_feat, freeze=False)
        self.text_trs = nn.Linear(self.t_feat.shape[1], self.feat_embed_dim)
        self.mm_adj = graph.build_freedom_mm_adj(self.v_feat, self.t_feat, self.knn_k, self.mm_image_weight)
        self.dropoutf = nn.Dropout(config["dropout"])

    def pre_epoch_processing(self):
        # degree-sensitive edge pruning, keep length int(nnz * 0.3) as the reference computes it
        self.sub_graph, _ = self.pruner.sample(keep_len=int(self.edge_values.size(0) * 0.3))

    def _item_embeds(self):
        image_feats = ops.project(self.image_embedding.weight, self.image_trs.weight, self.image_trs.bias, l2_normalize=True)
        text_feats = ops.project(self.text_embedding.weight, self.text_trs.weight, self.text_trs.bias, l2_normalize=True)
        return torch.cat([image_feats, text_feats], dim=1)

    def forward(self, adj):
        user_embeds = torch.cat([self.user_image.weight, self.user_text.weight], dim=1)
        item_embeds = self._item_embeds()
        if not torch.is_grad_enabled() and user_embeds.is_cuda and self.n_layers >= 1 and self.n_ui_layers >= 1:
            # inference: layer 1 reads the two tables in place, the item-item product shares its launch, `i_g + h` rides in
            # the last layer's epilogue
            all_emb = ops.propagate_mean_fused(adj, (user_embeds, item_embeds), self.n_ui_layers, post_csr=self.mm_adj,
                                               post_x=item_embeds, post_layers=self.n_layers, post_row0=self.n_users,
                                               cooperative=False)
            return torch.split(all_emb, [self.n_users, self.n_items], dim=0)
        ego = torch.cat((user_embeds, item_embeds), dim=0)
        all_emb = ops.propagate_mean(adj, ego, self.n_ui_layers)
        u_g, i_g = torch.split(all_emb, [self.n_users, self.n_items], dim=0)
        if self.n_layers == 0:
            return u_g, i_g + item_embeds
        h = item_embeds
        for _ in range(self.n_layers - 1):
            h = ops.spmm(self.mm_adj, h)
        return u_g, ops.spmm(self.mm_adj, h, base=i_g)           # i_g + mm_adj^n @ item_embeds, fused

    def _dropout_masks(self, B, d, device):
        """The masks of the reference's four `self.dropoutf` calls on [B, d] rows (views a, b of the users, c, d of the
        positive items, in that order), drawn by the call `nn.Dropout` makes -- `torch.native_dropout` on a fresh [B, d]
        tensor -- so the generator advances exactly as it does in the reference.  None where `nn.Dropout` draws nothing
        (p == 0 or eval mode); p == 1 drops everything without a draw."""
        p = float(self.dropoutf.p)
        if not self.training or p == 0.0:
            return None
        if p >= 1.0:
            return [torch.zeros(B, d, dtype=torch.bool, device=device) for _ in range(4)]
        src = torch.empty(B, d, dtype=torch.float32, device=device)
        return [torch.native_dropout(src, p, True)[1] for _ in range(4)]

    def calculate_loss(self, interaction):
        users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
        ua, ia = self.forward(self.sub_graph)
        masks = self._dropout_masks(users.numel(), ua.shape[1], ua.device)
        return ops.pgl_loss(ua, ia, users, pos_items, neg_items, masks, float(self.dropoutf.p), self.reg_weight)

    def _score_embeddings(self):
        return self._cached_eval_embeddings(lambda: self.forward(self.norm_adj))

    def full_sort_predict(self, interaction):
        u, i = self._score_embeddings()
        return ops.score(u, i, interaction[0])
