"""Worker of tests/test_itemknncbf_host.py: ItemKNNCBF (`mmrec_b200.models.itemknncbf`) under the harness of
tests/contract.py, with the kernels replaced by CPU stand-ins restated from tests/itemknncbf_oracle.py, against
tests/golden/itemknncbf_tiny.npz recorded from the reference's class."""
import sys

import numpy as np
import torch

import contract as C
import itemknncbf_oracle as KO

SHRINK = {"s10_": 10, "s0_": 0}


def _knn_arrays(S):
    """(values [I, k], indices [I, k]) of a kNN CSR stand-in (columns ascending per row)."""
    i, v = S.t_.indices(), S.t_.values()
    k = i.shape[1] // S.n_rows
    return v.reshape(S.n_rows, k).numpy(), i[1].reshape(S.n_rows, k).numpy()


def install():
    from mmrec_b200 import ops

    def knn_topk(x, k, rows=None, norms=None, shrink=None):         # K7's shrink route restated: itemknncbf.py:56-63, in
        assert rows is None and shrink is not None                   # float64 (no dependence on the CPU's fp32 GEMM)
        return KO.item_sim_topk_f64(x, k, shrink)

    def sparse_scores(R, S, users=None):                             # K9: the ordered sum
        r, c, v = R.coo()
        kv, ki = _knn_arrays(S)
        return torch.from_numpy(KO.ordered_scores(r.numpy(), c.numpy(), v.numpy(), R.n_rows, kv, ki,
                                                  users=None if users is None else users.numpy()))

    def sparse_score_topk(R, S, users, mask, k):                     # K9's ranking rule on the summed columns
        sc = sparse_scores(R, S, users).numpy()
        vals, idxs = [], []
        for b in range(sc.shape[0]):
            cols = np.nonzero(sc[b].view(np.uint32))[0]
            masked = [] if mask is None else mask[1][mask[0] == b].numpy()
            v, i = KO.sparse_rank(cols, sc[b][cols], masked, sc.shape[1], k)
            vals.append(v)
            idxs.append(i)
        return torch.from_numpy(np.stack(vals)), torch.from_numpy(np.stack(idxs))
    ops.knn_topk, ops.sparse_scores, ops.sparse_score_topk = knn_topk, sparse_scores, sparse_score_topk


def main(prefix):
    h = C.build("ItemKNNCBF", over={"shrink": [SHRINK[prefix]]}, install=install)
    model, sub = h.model, C.case(C.load("itemknncbf_tiny.npz"), prefix)
    kv, ki = _knn_arrays(model.item_sim)
    feats = KO.features(model.v_feat, model.t_feat)
    knn_ok, _ = KO.knn_agrees(kv, ki, sub["knn_val"], sub["knn_ind"], feats, SHRINK[prefix])
    sc = C.predict(model, sub)
    out = {"knn_ok": bool(knn_ok), "score_err": float(np.abs(sc - sub["scores"]).max() / np.abs(sub["scores"]).max()),
           "params": [k for k, _ in model.named_parameters()],
           "dummy_ok": bool(np.array_equal(model.dummy_embeddings.detach().numpy(), sub["dummy_embeddings"]))}
    out.update(C.check_metrics(h, sub))
    C.emit(out)


if __name__ == "__main__":
    main(sys.argv[1])
