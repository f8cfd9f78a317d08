"""Top-k evaluator with the reference's metric definitions (`src/utils/topk_evaluator.py:58-102`,
`src/utils/metrics.py:12-105`): Recall / NDCG / Precision / MAP at each k of `config['topk']`, averaged over
users, rounded to 4 decimals.  The hit matrix is built by a vectorised membership test instead of the reference's
O(U * k * |pos|) Python loop (SURVEY.md 8f f2)."""
import numpy as np
import torch


def hit_matrix(topk_index: np.ndarray, pos_items) -> np.ndarray:
    n_users, K = topk_index.shape
    lens = np.array([len(p) for p in pos_items], dtype=np.int64)
    if lens.sum() == 0:
        return np.zeros((n_users, K), dtype=bool)
    stride = int(max(topk_index.max(), max(int(p.max()) for p in pos_items if len(p))) + 1)
    keys = np.sort(np.repeat(np.arange(n_users, dtype=np.int64), lens) * stride + np.concatenate(pos_items).astype(np.int64))
    q = (np.arange(n_users, dtype=np.int64)[:, None] * stride + topk_index.astype(np.int64)).reshape(-1)
    pos = np.minimum(np.searchsorted(keys, q), len(keys) - 1)
    return (keys[pos] == q).reshape(n_users, K)


def recall_(hit, pos_len):
    return (np.cumsum(hit, axis=1) / pos_len.reshape(-1, 1)).mean(axis=0)


def recall2_(hit, pos_len):
    return np.cumsum(hit, axis=1).sum(axis=0) / pos_len.sum()


def precision_(hit, pos_len):
    return (hit.cumsum(axis=1) / np.arange(1, hit.shape[1] + 1)).mean(axis=0)


def ndcg_(hit, pos_len):
    K = hit.shape[1]
    disc = 1.0 / np.log2(np.arange(1, K + 1) + 1.0)
    idcg_all = np.cumsum(disc)
    # ideal DCG saturates once every positive is ranked: idcg[u, j] = idcg_all[min(j, min(pos_len, K) - 1)]
    cap = np.minimum(pos_len, K).astype(np.int64) - 1
    idcg = idcg_all[np.minimum(np.arange(K)[None, :], cap[:, None])]
    dcg = np.cumsum(np.where(hit, disc[None, :], 0.0), axis=1)
    return (dcg / idcg).mean(axis=0)


def map_(hit, pos_len):
    K = hit.shape[1]
    pre = hit.cumsum(axis=1) / np.arange(1, K + 1)
    sum_pre = np.cumsum(pre * hit.astype(float), axis=1)
    cap = np.minimum(pos_len, K).astype(np.int64)
    ranges = np.minimum(np.arange(1, K + 1)[None, :], cap[:, None])
    return (sum_pre / ranges).mean(axis=0)


metrics_dict = {"ndcg": ndcg_, "recall": recall_, "recall2": recall2_, "precision": precision_, "map": map_}


class TopKEvaluator(object):
    def __init__(self, config):
        self.config = config
        self.metrics = [m.lower() for m in ([config["metrics"]] if isinstance(config["metrics"], str) else config["metrics"])]
        self.topk = [config["topk"]] if isinstance(config["topk"], int) else list(config["topk"])
        for m in self.metrics:
            if m not in metrics_dict:
                raise ValueError("There is no user grouped topk metric named {}!".format(m))
        for k in self.topk:
            if k <= 0:
                raise ValueError("topk must be a positive integer or a list of positive integers, but get `{}`".format(k))

    def _evaluate_on_device(self, batch_matrix_list, eval_data):
        """f2: the hit matrix and the metric sums are computed where the index matrix lives (`mmrec_topk_metrics_f64`);
        4 x K float64 sums come back instead of the [n_users, K] matrix.  `recall2` (a ratio of sums over users) and
        K > 128 take the host route."""
        from .. import ops
        dev = batch_matrix_list[0].device
        cache = getattr(eval_data, "_pos_csr_dev", None)
        if cache is None or cache[0] != dev:
            pos = eval_data.get_eval_items()
            lens = np.array([len(p) for p in pos], dtype=np.int64)
            ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
            items = np.concatenate([np.sort(np.asarray(p, dtype=np.int64)) for p in pos]) if len(pos) else np.zeros(0, np.int64)
            cache = (dev, torch.from_numpy(ptr).to(dev), torch.from_numpy(items).to(dev))
            eval_data._pos_csr_dev = cache
        _, ptr, items = cache
        K = batch_matrix_list[0].shape[1]
        disc = 1.0 / np.log2(np.arange(1, K + 1) + 1.0)
        disc_d, idcg_d = torch.from_numpy(disc).to(dev), torch.from_numpy(np.cumsum(disc)).to(dev)
        sums = torch.zeros(4, K, dtype=torch.float64, device=dev)
        row = 0
        for m in batch_matrix_list:
            m = m.contiguous()
            ops.topk_metric_sums(m, ptr[row:row + m.shape[0] + 1], items, disc_d, idcg_d, sums)
            row += m.shape[0]
        assert row == ptr.numel() - 1
        mean = (sums / row).cpu().numpy()
        rows = {"recall": 0, "ndcg": 1, "precision": 2, "map": 3}
        return {"{}@{}".format(m, k): round(float(mean[rows[m], k - 1]), 4) for m in self.metrics for k in self.topk}

    def evaluate(self, batch_matrix_list, eval_data, is_test=False, idx=0):
        if (len(batch_matrix_list) and batch_matrix_list[0].is_cuda and batch_matrix_list[0].shape[1] <= 128
                and all(m in ("recall", "ndcg", "precision", "map") for m in self.metrics)
                and self.config["device_evaluator"] is not False):
            return self._evaluate_on_device(batch_matrix_list, eval_data)
        pos_items = eval_data.get_eval_items()
        pos_len = np.asarray(eval_data.get_eval_len_list())
        topk_index = torch.cat(batch_matrix_list, dim=0).cpu().numpy()
        assert len(pos_len) == len(topk_index)
        hit = hit_matrix(topk_index, pos_items)
        out = {}
        for m in self.metrics:
            v = metrics_dict[m](hit, pos_len)
            for k in self.topk:
                out["{}@{}".format(m, k)] = round(float(v[k - 1]), 4)
        return out
