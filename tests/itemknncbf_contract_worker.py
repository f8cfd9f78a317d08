"""Worker of tests/test_itemknncbf_host.py (own process: the kernels behind `mmrec_b200.ops` are patched).

ItemKNNCBF (`mmrec_b200.models.itemknncbf`) under the harness of tests/dropin_contract_worker.py -- built the way
quick_start builds it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels
replaced by CPU stand-ins restated from tests/itemknncbf_oracle.py, against tests/golden/itemknncbf_tiny.npz recorded from the
reference's class."""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import itemknncbf_oracle as KO  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402

SHRINK = {"s10_": 10, "s0_": 0}


def _knn_arrays(S):
    """(values [I, k], indices [I, k]) of a kNN CSR stand-in (columns ascending per row)."""
    i, v = S.t_.indices(), S.t_.values()
    k = i.shape[1] // S.n_rows
    return v.reshape(S.n_rows, k).numpy(), i[1].reshape(S.n_rows, k).numpy()


def install_itemknncbf_ops():
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
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    config = Config("ItemKNNCBF", "tiny", dict({"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512,
                                                "shrink": [SHRINK[prefix]]}, **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    dataset = RecDataset(config)
    str(dataset)
    tr, va, te = dataset.split()
    str(tr), str(va), str(te)
    train_data = TrainDataLoader(config, tr, batch_size=config["train_batch_size"], shuffle=True)
    valid_data = EvalDataLoader(config, va, additional_dataset=tr, batch_size=config["eval_batch_size"])
    test_data = EvalDataLoader(config, te, additional_dataset=tr, batch_size=config["eval_batch_size"])
    init_seed(config["seed"])
    train_data.pretrain_setup()
    install_cpu_ops()
    install_itemknncbf_ops()
    from mmrec_b200.models.itemknncbf import ItemKNNCBF
    model = ItemKNNCBF(config, train_data).to(config["device"])
    gold = np.load(os.path.join(HERE, "golden", "itemknncbf_tiny.npz"), allow_pickle=True)
    G = lambda k: gold[prefix + k]
    kv, ki = _knn_arrays(model.item_sim)
    feats = KO.features(model.v_feat, model.t_feat)
    knn_ok, _ = KO.knn_agrees(kv, ki, G("knn_val"), G("knn_ind"), feats, SHRINK[prefix])
    model.eval()
    with torch.no_grad():
        sc = model.full_sort_predict([torch.from_numpy(G("eval_users")), torch.from_numpy(G("eval_mask"))])
    score_err = float(np.abs(sc.numpy() - G("scores")).max() / np.abs(G("scores")).max())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in G("metric_names")]
    out = {"knn_ok": bool(knn_ok), "score_err": score_err,
           "params": [k for k, _ in model.named_parameters()],
           "dummy_ok": bool(np.array_equal(model.dummy_embeddings.detach().numpy(), G("dummy_embeddings"))),
           "valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in G("metric_values")])),
           "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in G("test_metric_values")]))}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    main(sys.argv[1])
