"""Worker of tests/test_grcn_contract.py (own process: the kernels behind `mmrec_b200.ops` are patched).

GRCN (`mmrec_b200.models.grcn`) under the harness of tests/dropin_contract_worker.py -- built the way quick_start builds
it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by
`install_cpu_ops`'s CPU stand-ins plus three for GRCN: the attention graph as its COO in `graph.grcn_edge_order`'s order,
`ops.edge_attention` as PyG's gathers, grouped softmax and `index_add_`, and `ops.spmm_values` as a gather and
`index_add_`.  Against tests/golden/grcn_tiny.npz / traj_grcn_tiny.npz recorded from the reference's class."""
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

import dualgnn_golden as G  # noqa: E402
from make_golden_grcn import CASES, TRAJ_LR, softmax  # noqa: E402
import selfcf_golden  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402


class _AttnGraph:
    """What GRCN reads of its attention CSR: the entries in CSR order."""

    def __init__(self, rows, cols, n):
        self.rows, self.cols, self.n_rows, self.n_cols = rows, cols, n, n
        self.colidx, self.nnz = cols, rows.numel()


def install_grcn_ops():
    from mmrec_b200 import graph, ops

    def build_grcn_adj(inter, n_users, n_items, device):
        rows, cols, order = graph.grcn_edge_order(inter.row, inter.col, n_users, n_items)
        return _AttnGraph(torch.from_numpy(rows), torch.from_numpy(cols), n_users + n_items), torch.from_numpy(order)
    graph.build_grcn_adj = build_grcn_adj

    def edge_attention(A, X, base=None):
        alpha = softmax((X[A.rows] * X[A.cols]).sum(-1), A.rows, num_nodes=A.n_rows)
        Y = torch.zeros_like(X).index_add_(0, A.rows, X[A.cols] * alpha.view(-1, 1))
        return (Y if base is None else base + Y), alpha
    ops.edge_attention = edge_attention
    ops.spmm_values = lambda A, vals, X: torch.zeros_like(X).index_add_(0, A.rows, X[A.cols] * vals.view(-1, 1))


def _setup(epochs=None, image_only=False, overrides=None):
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, None if image_only else t)
    over = {"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}
    config = Config("GRCN", "tiny", dict(over, **extra, **(overrides or {})))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    if epochs:
        config["epochs"] = epochs
        config["learning_rate"] = TRAJ_LR
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
    install_grcn_ops()
    from mmrec_b200.models.grcn import GRCN
    model = GRCN(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def main_model(p=""):
    over, mods = CASES[p]
    config, model, valid_data, test_data, Trainer = _setup(image_only=mods == "v", overrides=dict(over))
    gold = np.load(os.path.join(HERE, "golden", "grcn_tiny.npz"), allow_pickle=True)
    sub = {k[len(p):]: gold[k] for k in gold.files
           if k.startswith(p) and not any(k.startswith(q) for q in CASES if q and q != p and len(q) > len(p))}
    init = {k: v for k, v in sub.items() if k.startswith("init_sha256.")}

    class _G:
        files = list(init)

        def __getitem__(self, k):
            return init[k]
    out = {"init_identical": not selfcf_golden.same_init(model, _G())
           and [k for k, _ in model.named_parameters()] == [str(x) for x in sub["param_order"]]
           and G.equal(sub, "rng_after_init", torch.get_rng_state().numpy())}
    eb = [torch.from_numpy(sub["eval_users"]), torch.from_numpy(sub["eval_mask"])]
    model.eval()
    with torch.no_grad():
        out["pre_score_rel"] = G.rel(sub, "pre.scores", model.full_sort_predict(eb).numpy())
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(sub["batch"]))
    out["representation_rel"] = G.rel(sub, "representation", model.result.detach().numpy())
    loss.backward()
    named = dict(model.named_parameters())
    grads = [k[5:] for k in G.recorded(sub, "grad.")]
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0]), "loss_shape": list(loss.shape),
                "grad_keys": sorted(k for k, q in named.items() if q.grad is not None) == grads,
                "grad_rel": {k: G.rel(sub, "grad." + k, named[k].grad.numpy()) for k in grads}})
    model.zero_grad()
    model.eval()
    with torch.no_grad():
        out["score_rel"] = G.rel(sub, "scores", model.full_sort_predict(eb).numpy())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in sub["metric_names"]]
    out.update({"valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in sub["metric_values"]])),
                "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in sub["test_metric_values"]]))})
    print("CONTRACT " + json.dumps(out))


def main_traj():
    config, model, valid_data, test_data, Trainer = _setup(epochs=2)
    gold = np.load(os.path.join(HERE, "golden", "traj_grcn_tiny.npz"), allow_pickle=True)
    trainer = Trainer(config, model)
    rec = {"losses": [], "valid": [], "test": []}
    orig = model.calculate_loss

    def spy(interaction):
        l = orig(interaction)
        rec["losses"].append(float(l.detach()))
        return l
    model.calculate_loss = spy
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    first = np.concatenate([[0], np.cumsum(gold["batches_per_epoch"])])
    batches = gold["batches"]
    recorded = [[torch.from_numpy(batches[:, offs[b]:offs[b + 1]].copy()) for b in range(first[ep], first[ep + 1])]
                for ep in range(len(gold["batches_per_epoch"]))]
    for ep in range(2):
        model.pre_epoch_processing()
        trainer._train_epoch(recorded[ep], ep)
        trainer.lr_scheduler.step()
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    out = {"n_batches": len(rec["losses"]), "want_batches": int(gold["n_steps"]),
           "loss_max_rel": float(np.max(np.abs(np.array(rec["losses"]) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(rec["valid"]) - gold["valid"]).max(), np.abs(np.array(rec["test"]) - gold["test"]).max()))}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    {"traj": main_traj, "l1": lambda: main_model("l1."), "image": lambda: main_model("image.")}.get(arg, main_model)()
