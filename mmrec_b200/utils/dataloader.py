"""Batch producers with the reference's output formats (`src/utils/dataloader.py`), vectorised.

* `TrainDataLoader` yields `LongTensor[3, B]` (user, positive, sampled negative) -- `[2, B]` when
  `use_neg_sampling` is False (`dataloader.py:226-260`).  The reference draws negatives one Python
  `random.sample` at a time with rejection (`:267-275`); here rejection sampling runs on whole numpy batches, so
  the sample distribution is the same (uniform over train items not in the user's history) but the random
  stream is not (SURVEY.md 8f f3).
* `EvalDataLoader` yields `[users LongTensor[<=B], mask LongTensor[2, nnz]]` with mask row = position inside the
  batch and column = train-positive item, grouped by user in batch order (`:359-391`), built from a CSR of the
  training interactions instead of per-user `groupby.get_group` loops.
* `inter_matrix(form)` returns the scipy COO/CSR of the training interactions (`:155-210`).
"""
import math

import numpy as np
import torch
from scipy.sparse import coo_matrix


class AbstractDataLoader(object):
    def __init__(self, config, dataset, additional_dataset=None, batch_size=1, neg_sampling=False, shuffle=False):
        self.config = config
        self.dataset = dataset
        self.dataset_bk = dataset.copy(dataset.df)
        self.additional_dataset = additional_dataset
        self.batch_size = self.step = batch_size
        self.shuffle = shuffle
        self.neg_sampling = neg_sampling
        self.device = config["device"]
        self.pr = 0
        self.inter_pr = 0

    def pretrain_setup(self):
        pass

    def __len__(self):
        return math.ceil(self.pr_end / self.step)

    def __iter__(self):
        if self.shuffle:
            self._shuffle()
        return self

    def __next__(self):
        if self.pr >= self.pr_end:
            self.pr = 0
            self.inter_pr = 0
            raise StopIteration()
        return self._next_batch_data()


class TrainDataLoader(AbstractDataLoader):
    def __init__(self, config, dataset, batch_size=1, shuffle=False):
        super().__init__(config, dataset, batch_size=batch_size, neg_sampling=True, shuffle=shuffle)
        df = dataset.df
        self.uid, self.iid = dataset.uid_field, dataset.iid_field
        self.all_items = np.sort(df[self.iid].unique())
        self.n_items = dataset.item_num
        from ..graph import unique_sorted
        self._hist_keys = unique_sorted(df[self.uid].values.astype(np.int64) * self.n_items + df[self.iid].values.astype(np.int64))
        self.use_neg = bool(config["use_neg_sampling"])
        self.rng = np.random.default_rng(0)

    def pretrain_setup(self):
        if self.shuffle:
            self.dataset = self.dataset_bk.copy(self.dataset_bk.df)
        seed = self.config["seed"]
        self.rng = np.random.default_rng(seed if isinstance(seed, int) else 0)

    def inter_matrix(self, form="coo", value_field=None):
        df = self.dataset.df
        src, tgt = df[self.uid].values, df[self.iid].values
        data = np.ones(len(df)) if value_field is None else df[value_field].values
        mat = coo_matrix((data, (src, tgt)), shape=(self.dataset.user_num, self.dataset.item_num))
        if form == "coo":
            return mat
        if form == "csr":
            return mat.tocsr()
        raise NotImplementedError("sparse matrix format [{}] has not been implemented.".format(form))

    @property
    def pr_end(self):
        return len(self.dataset)

    def _shuffle(self):
        self.dataset.shuffle()

    def _sample_neg(self, users: np.ndarray) -> np.ndarray:
        neg = self.all_items[self.rng.integers(0, len(self.all_items), users.shape[0])]
        while True:
            key = users * self.n_items + neg
            pos = np.searchsorted(self._hist_keys, key)
            bad = (pos < len(self._hist_keys)) & (self._hist_keys[np.minimum(pos, len(self._hist_keys) - 1)] == key)
            n_bad = int(bad.sum())
            if n_bad == 0:
                return neg
            neg[bad] = self.all_items[self.rng.integers(0, len(self.all_items), n_bad)]

    def _next_batch_data(self):
        cur = self.dataset[self.pr: self.pr + self.step]
        self.pr += self.step
        users = cur[self.uid].values.astype(np.int64)
        items = cur[self.iid].values.astype(np.int64)
        rows = [users, items]
        if self.use_neg:
            rows.append(self._sample_neg(users))
        return torch.from_numpy(np.stack(rows)).to(self.device)


class EvalDataLoader(AbstractDataLoader):
    def __init__(self, config, dataset, additional_dataset=None, batch_size=1, shuffle=False):
        super().__init__(config, dataset, additional_dataset=additional_dataset, batch_size=batch_size, shuffle=shuffle)
        if additional_dataset is None:
            raise ValueError("Training datasets is nan")
        uid, iid = dataset.uid_field, dataset.iid_field
        eval_u = dataset.df[uid].unique()                       # order of first appearance, like the reference
        tr = additional_dataset.df
        tr_u, tr_i = tr[uid].values.astype(np.int64), tr[iid].values.astype(np.int64)
        order = np.argsort(tr_u, kind="stable")                 # per-user items keep their order of appearance
        ptr = np.zeros(dataset.user_num + 1, dtype=np.int64)
        np.add.at(ptr, tr_u + 1, 1)
        ptr = np.cumsum(ptr)
        lens = ptr[eval_u + 1] - ptr[eval_u]
        if (lens == 0).any():
            raise KeyError("evaluation user without training interactions")
        self.train_pos_len_list = lens.tolist()
        starts = np.repeat(ptr[eval_u], lens)
        within = np.arange(lens.sum()) - np.repeat(np.cumsum(lens) - lens, lens)
        self._mask_items = tr_i[order][starts + within]
        self._mask_users = np.repeat(np.arange(len(eval_u)), lens)
        self._mask_ptr = np.concatenate([[0], np.cumsum(lens)])
        self.pos_items_per_u = torch.from_numpy(np.stack([self._mask_users, self._mask_items])).to(self.device)
        # ground truth per eval user
        ev_u, ev_i = dataset.df[uid].values.astype(np.int64), dataset.df[iid].values.astype(np.int64)
        eorder = np.argsort(ev_u, kind="stable")
        eptr = np.zeros(dataset.user_num + 1, dtype=np.int64)
        np.add.at(eptr, ev_u + 1, 1)
        eptr = np.cumsum(eptr)
        sorted_items = ev_i[eorder]
        self.eval_items_per_u = [sorted_items[eptr[u]:eptr[u + 1]] for u in eval_u]
        self.eval_len_list = (eptr[eval_u + 1] - eptr[eval_u]).astype(np.int64)
        self.eval_u = torch.from_numpy(eval_u.astype(np.int64)).to(self.device)

    @property
    def pr_end(self):
        return self.eval_u.shape[0]

    def _shuffle(self):
        self.dataset.shuffle()

    def _next_batch_data(self):
        lo, hi = self.pr, min(self.pr + self.step, self.pr_end)
        users = self.eval_u[lo:hi]
        a, b = int(self._mask_ptr[lo]), int(self._mask_ptr[hi])
        mask = self.pos_items_per_u[:, a:b].clone()
        mask[0] -= lo
        self.inter_pr = b
        self.pr += self.step
        return [users, mask]

    def get_eval_items(self):
        return self.eval_items_per_u

    def get_eval_len_list(self):
        return self.eval_len_list

    def get_eval_users(self):
        return self.eval_u.cpu()
