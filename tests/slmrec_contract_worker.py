"""Worker of tests/test_slmrec_contract.py (own process: the kernels behind `mmrec_b200.ops` are patched).

SLMRec (`mmrec_b200.models.slmrec`) under the harness of tests/dropin_contract_worker.py -- built the way quick_start builds
it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by
`install_cpu_ops`'s CPU stand-ins (`ops.project` = `F.linear`, `ops.propagate_mean` = `torch.sparse.mm` + stack + mean on
the [N, 3d] ego table, `ops.score` = the dense product), against tests/golden/slmrec_tiny.npz / traj_slmrec_tiny.npz
recorded from the reference's class."""
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

import selfcf_golden  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402


def _setup(epochs=None):
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    over = {"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}
    config = Config("SLMRec", "tiny", dict(over, **extra))
    config["inter_file_name"] = "tiny.inter"
    config["USER_ID_FIELD"], config["ITEM_ID_FIELD"] = "userID", "itemID"
    config["vision_feature_file"], config["text_feature_file"] = "image_feat.npy", "text_feat.npy"
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
    from mmrec_b200.models.slmrec import SLMRec
    model = SLMRec(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / max(np.linalg.norm(b), 1e-30))


def main_model():
    config, model, valid_data, test_data, Trainer = _setup()
    gold = np.load(os.path.join(HERE, "golden", "slmrec_tiny.npz"), allow_pickle=True)
    out = {"init_identical": not selfcf_golden.same_init(model, gold)
           and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]}
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    out["views_equal"] = {n: bool(np.array_equal(getattr(model, n).detach().numpy(), gold["view_" + n])) for n in ("i_emb", "v_emb", "t_emb")}
    out["tables_equal"] = bool(np.array_equal(model.all_users.detach().numpy(), gold["all_users"])
                               and np.array_equal(model.all_items.detach().numpy(), gold["all_items"]))
    loss.backward()
    named = dict(model.named_parameters())
    grads = {k[5:]: gold[k] for k in gold.files if k.startswith("grad.")}
    out.update({"loss": float(loss.item()), "want_loss": float(gold["loss"][0]),
                "grad_keys": sorted(k for k, p in named.items() if p.grad is not None) == sorted(grads),
                "grad_rel": {k: rel(named[k].grad.numpy(), g) for k, g in grads.items()},
                "grad_equal": sorted(k for k, g in grads.items() if np.array_equal(named[k].grad.numpy(), g))})
    model.zero_grad()
    model.eval()
    with torch.no_grad():
        sc = model.full_sort_predict([torch.from_numpy(gold["eval_users"]), torch.from_numpy(gold["eval_mask"])])
    out["score_equal"] = bool(np.array_equal(sc.numpy(), gold["scores"]))
    out["score_err"] = float(np.abs(sc.numpy() - gold["scores"]).max())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in gold["metric_names"]]
    out.update({"valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in gold["metric_values"]])),
                "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in gold["test_metric_values"]]))})
    print("CONTRACT " + json.dumps(out))


def main_traj():
    config, model, valid_data, test_data, Trainer = _setup(epochs=2)
    gold = np.load(os.path.join(HERE, "golden", "traj_slmrec_tiny.npz"), allow_pickle=True)
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
    recorded = [[torch.from_numpy(gold["batches"][:, offs[b]:offs[b + 1]]) for b in range(first[ep], first[ep + 1])]
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
    {"traj": main_traj}.get(sys.argv[1] if len(sys.argv) > 1 else "", main_model)()
