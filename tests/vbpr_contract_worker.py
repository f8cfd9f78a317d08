"""Worker of tests/test_vbpr_contract.py (own process: the kernels behind `mmrec_b200.ops` are patched).

VBPR and BPR (`mmrec_b200.models.vbpr`, `.bpr`) under the harness of tests/dropin_contract_worker.py -- built the way
quick_start builds them, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the
kernels replaced by `install_cpu_ops`'s CPU stand-ins plus one for `ops.bpr_mf_loss`, the reference's torch expression on
the gathered rows (vbpr_golden.torch_bpr_mf_loss), against tests/golden/{vbpr,bpr}_tiny.npz and traj_{vbpr,bpr}_tiny.npz
recorded from the reference's classes."""
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
import selfcf_golden  # noqa: E402
import vbpr_golden as V  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402


def _setup(name, mods, epochs=None):
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", synth.make_graph(u, i, e, seed=0), v if "v" in mods else None, t if "t" in mods else None)
    config = Config(name, "tiny", dict({"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}, **extra))
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
    from mmrec_b200 import ops
    ops.bpr_mf_loss = V.torch_bpr_mf_loss
    from mmrec_b200.utils.utils import get_model
    model = get_model(name)(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def main_model(p):
    name, mods = V.CASES[p]
    config, model, valid_data, test_data, Trainer = _setup(name, mods)
    gold = np.load(os.path.join(HERE, "golden", f"{name.lower()}_tiny.npz"), allow_pickle=True)
    sub = {k[len(p):]: gold[k] for k in gold.files if k.startswith(p)}
    init = {k[len("init_sha256."):]: str(v) for k, v in sub.items() if k.startswith("init_sha256.")}
    out = {"init_identical": selfcf_golden.init_digests(model) == init
           and [k for k, _ in model.named_parameters()] == [str(x) for x in sub["param_order"]]
           and G.equal(sub, "rng_after_init", torch.get_rng_state().numpy())}
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(sub["batch"]))
    loss.backward()
    named = dict(model.named_parameters())
    grads = [k[5:] for k in G.recorded(sub, "grad.")]
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0]), "loss_shape": list(loss.shape),
                "grad_keys": sorted(k for k, q in named.items() if q.grad is not None) == sorted(grads),
                "grad_rel": {k: G.rel(sub, "grad." + k, named[k].grad.numpy()) for k in grads}})
    model.zero_grad()
    model.eval()
    eb = [torch.from_numpy(sub["eval_users"]), torch.from_numpy(sub["eval_mask"])]
    with torch.no_grad():
        out["score_rel"] = G.rel(sub, "scores", model.full_sort_predict(eb).numpy())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in sub["metric_names"]]
    out["metric_max_abs"] = max(max(abs(valid[k] - w) for k, w in zip(names, sub["metric_values"])),
                                max(abs(test[k] - w) for k, w in zip(names, sub["test_metric_values"])))
    print("CONTRACT " + json.dumps(out))


def main_traj(name):
    config, model, valid_data, test_data, Trainer = _setup(name, V.TRAJ[name], epochs=2)
    gold = np.load(os.path.join(HERE, "golden", f"traj_{name.lower()}_tiny.npz"), allow_pickle=True)
    trainer = Trainer(config, model)
    rec = {"losses": [], "valid": [], "test": [], "rng_kept": []}
    orig = model.calculate_loss

    def spy(interaction):
        st = torch.get_rng_state()
        l = orig(interaction)
        rec["rng_kept"].append(bool(torch.equal(st, torch.get_rng_state())))
        rec["losses"].append(float(l.detach()))
        return l
    model.calculate_loss = spy
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    first = np.concatenate([[0], np.cumsum(gold["batches_per_epoch"])])
    recorded = [[torch.from_numpy(gold["batches"][:, offs[b]:offs[b + 1]].copy()) for b in range(first[ep], first[ep + 1])]
                for ep in range(len(gold["batches_per_epoch"]))]
    for ep in range(2):
        model.pre_epoch_processing()
        trainer._train_epoch(recorded[ep], ep)
        trainer.lr_scheduler.step()
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    out = {"n_batches": len(rec["losses"]), "want_batches": int(gold["n_steps"]),
           "rng_kept": all(rec["rng_kept"]) and bool(np.all(gold["rng_kept"])),
           "loss_max_rel": float(np.max(np.abs(np.array(rec["losses"]) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(rec["valid"]) - gold["valid"]).max(), np.abs(np.array(rec["test"]) - gold["test"]).max()))}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    arg = sys.argv[1]
    main_traj(arg[5:]) if arg.startswith("traj:") else main_model(arg)
