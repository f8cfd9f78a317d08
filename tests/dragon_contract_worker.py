"""Worker of tests/test_dragon_contract.py (own process: the kernels behind `mmrec_b200.ops` are patched).

DRAGON (`mmrec_b200.models.dragon`) under the harness of tests/dropin_contract_worker.py -- built the way quick_start
builds it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by
`install_cpu_ops`'s CPU stand-ins plus one for `ops.propagate_sum` (the reference's `h = A x`, `h_1 = A h`, `h + x + h_1`
with `torch.sparse.mm`), against tests/golden/dragon_tiny.npz / traj_dragon_tiny.npz recorded from the reference's class.
The dataset's `user_graph_dict.npy` is written by `synth.write_user_graph_dict`."""
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
from make_golden_dragon import CASES  # noqa: E402
import selfcf_golden  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402


def _setup(epochs=None, text_only=False, overrides=None):
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, None if text_only else v, t)
    synth.write_user_graph_dict(data, "tiny", g)
    over = {"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}
    config = Config("DRAGON", "tiny", dict(over, **extra, **(overrides or {})))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
    config["user_graph_dict_file"] = "user_graph_dict.npy"
    for k in config["hyper_parameters"]:
        if isinstance(config[k], list):
            config[k] = config[k][0]
    if epochs:
        config["epochs"] = epochs
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
    from mmrec_b200 import ops

    def propagate_sum(A, ego, n_layers):
        out, x = ego, ego
        for _ in range(n_layers):
            x = torch.sparse.mm(A.t_, x)
            out = x + out if out is ego else out + x                     # (h + x) + h_1, dualgnn.py:314
        return out
    ops.propagate_sum = propagate_sum

    from mmrec_b200.models.dragon import DRAGON
    model = DRAGON(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def user_rep(model):
    """`user_rep` before the user graph, from the towers' outputs the forward kept (`v_rep` / `t_rep`, dragon.py:231-243)."""
    U = model.n_users
    if model.v_rep is not None and model.t_rep is not None:
        w = model.weight_u.detach()
        return torch.cat((model.v_rep[:U, :, 0] * w[:, 0], model.t_rep[:U, :, 0] * w[:, 1]), dim=1).detach()
    return (model.t_rep if model.t_rep is not None else model.v_rep)[:U].detach()


def main_model(p=""):
    over, text_only = CASES[p]
    config, model, valid_data, test_data, Trainer = _setup(text_only=text_only, overrides={k: [v] for k, v in over.items()})
    gold = np.load(os.path.join(HERE, "golden", "dragon_tiny.npz"), allow_pickle=True)
    sub = {k[len(p):]: gold[k] for k in gold.files if k.startswith(p)} if p else {k: gold[k] for k in gold.files}
    init = {k: v for k, v in sub.items() if k.startswith("init_sha256.")}

    class _G:
        files = list(init)

        def __getitem__(self, k):
            return init[k]
    out = {"init_identical": not selfcf_golden.same_init(model, _G())
           and [k for k, _ in model.named_parameters()] == [str(x) for x in sub["param_order"]]
           and G.sha256(model.result_embed.numpy()) == str(sub["result_embed0_sha256"]),
           "has_v_gcn": hasattr(model, "v_gcn")}
    eb = [torch.from_numpy(sub["eval_users"]), torch.from_numpy(sub["eval_mask"])]
    model.eval()
    with torch.no_grad():
        s0 = model.full_sort_predict(eb)
    out["scores0_equal"] = bool(s0.dtype == torch.float64 and G.equal(sub, "scores0", s0.numpy()))
    np.random.seed(G.SAMPLE_SEED)
    model.pre_epoch_processing()
    out["sample_equal"] = bool(G.equal(sub, "sample_idx", model.epoch_user_graph.numpy())
                               and G.equal(sub, "sample_w", model.user_weight_matrix.numpy()))
    model.train()
    model.zero_grad()
    b = torch.from_numpy(sub["batch"]).clone()
    loss = model.calculate_loss(b)
    out["batch_after_equal"] = bool(np.array_equal(b.numpy(), sub["batch_after"]))
    out["user_rep_rel"] = G.rel(sub, "user_rep", user_rep(model).numpy())
    out["result_embed_rel"] = G.rel(sub, "result_embed", model.result_embed.detach().numpy())
    loss.backward()
    named = dict(model.named_parameters())
    grads = [k[5:] for k in G.recorded(sub, "grad.")]
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0]),
                "grad_keys": sorted(k for k, q in named.items() if q.grad is not None) == grads,
                "grad_rel": {k: G.rel(sub, "grad." + k, named[k].grad.numpy()) for k in grads}})
    model.zero_grad()
    model.eval()
    with torch.no_grad():
        sc = model.full_sort_predict(eb)
    out["score_rel"] = G.rel(sub, "scores", sc.numpy())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in sub["metric_names"]]
    out.update({"valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in sub["metric_values"]])),
                "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in sub["test_metric_values"]]))})
    print("CONTRACT " + json.dumps(out))


def main_traj():
    config, model, valid_data, test_data, Trainer = _setup(epochs=2)
    gold = np.load(os.path.join(HERE, "golden", "traj_dragon_tiny.npz"), allow_pickle=True)
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
        np.random.seed(int(gold["epoch_seed0"]) + ep)
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
    {"traj": main_traj, "text": lambda: main_model("text."), "mean": lambda: main_model("mean.")}.get(arg, main_model)()
