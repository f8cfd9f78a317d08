"""Model-side boundary of the hot path: the class contract the reference's trainer drives.

Mirrors `src/common/abstract_recommender.py:10-103` (same method names, attributes and config
keys) so that the model classes in `mmrec_b200.models` are drop-ins under the reference's `src/models`
(see INTEGRATION.md).  Extra, optional entry point used by this repo's trainer:
`full_sort_topk(interaction, k)` -- the fused scoring + mask + top-k fast path.
"""
import os

import numpy as np
import torch
import torch.nn as nn


class AbstractRecommender(nn.Module):
    def pre_epoch_processing(self):
        pass

    def post_epoch_processing(self):
        pass

    def calculate_loss(self, interaction):
        raise NotImplementedError

    def predict(self, interaction):
        raise NotImplementedError

    def full_sort_predict(self, interaction):
        raise NotImplementedError

    def __str__(self):
        n_params = sum(int(np.prod(p.size())) for p in self.parameters())
        return super().__str__() + "\nTrainable parameters: {}".format(n_params)


class GeneralRecommender(AbstractRecommender):
    """Reads the dataset sizes and the pre-extracted modality features exactly like the reference
    (`abstract_recommender.py:75-103`): `image_feat.npy` / `text_feat.npy` under `data_path + dataset`,
    fp32, moved to `config['device']`."""

    def __init__(self, config, dataloader):
        super().__init__()
        self.USER_ID = config["USER_ID_FIELD"]
        self.ITEM_ID = config["ITEM_ID_FIELD"]
        self.NEG_ITEM_ID = config["NEG_PREFIX"] + self.ITEM_ID
        self.n_users = dataloader.dataset.get_user_num()
        self.n_items = dataloader.dataset.get_item_num()
        self.batch_size = config["train_batch_size"]
        self.device = config["device"]
        self.v_feat, self.t_feat = None, None
        if not config["end2end"] and config["is_multimodal_model"]:
            root = os.path.abspath(config["data_path"] + config["dataset"])
            vp = os.path.join(root, config["vision_feature_file"])
            tp = os.path.join(root, config["text_feature_file"])
            if os.path.isfile(vp):
                self.v_feat = torch.from_numpy(np.load(vp, allow_pickle=True)).type(torch.FloatTensor).to(self.device)
            if os.path.isfile(tp):
                self.t_feat = torch.from_numpy(np.load(tp, allow_pickle=True)).type(torch.FloatTensor).to(self.device)
            assert self.v_feat is not None or self.t_feat is not None, "Features all NONE"
        self._eval_cache = None

    # ---- shared helpers for the graph models --------------------------------------------------------
    def _cached_eval_embeddings(self, compute):
        """`full_sort_predict` re-runs the whole propagation for every eval batch in the reference
        (`freedom.py:215`), although the embeddings cannot change inside `Trainer.evaluate`.  Under eval + no_grad the
        result (and the packed item operand of the fused top-k, `ops.Catalog`) is kept while nothing it depends on
        changes: the key holds the version counter of every parameter and buffer (optimizer steps, `load_state_dict`,
        in-place edits all bump it) and the identity of the graph attributes a model names in `_eval_cache_deps`
        (`norm_adj`, `masked_adj`, ...).  Bit-identical to recomputing; removes the largest item of
        `full_sort_predict` (SURVEY.md 3.4).  (Writes through `.data` bypass version counters: call `train()`/`eval()`
        or `invalidate_eval_cache()` after such an edit.)"""
        if self.training or torch.is_grad_enabled():
            return compute()
        key = (tuple((id(t), t._version) for t in self.parameters()) + tuple((id(t), t._version) for t in self.buffers()),
               tuple(id(getattr(self, a, None)) for a in self._eval_cache_deps))
        if self._eval_cache is None or self._eval_cache[0] != key:
            self._eval_cache = (key, compute(), None)
        return self._eval_cache[1]

    _eval_cache_deps = ("norm_adj", "masked_adj", "forward_adj", "mm_adj", "image_adj", "text_adj", "R")

    def invalidate_eval_cache(self):
        self._eval_cache = None

    def train(self, mode: bool = True):
        self._eval_cache = None
        return super().train(mode)

    def full_sort_topk(self, interaction, k):
        """Fused `full_sort_predict` + `scores[mask] = -1e10` + `torch.topk(scores, k)`
        (`src/common/trainer.py:304-309`); returns the index matrix only, like the trainer keeps."""
        from .. import ops
        u, i = self._score_embeddings()
        cat = None
        c = self._eval_cache
        if c is not None and c[1][1] is i and i.shape[1] <= 128:       # cached embeddings: their item operand is packed once
            if c[2] is None:
                self._eval_cache = c = (c[0], c[1], ops.Catalog(i))
            cat, i = c[2], c[2].item_e
        _, idx = ops.score_topk(u, i, interaction[0], interaction[1], k, catalog=cat)
        return idx

    def _score_embeddings(self):
        raise NotImplementedError
