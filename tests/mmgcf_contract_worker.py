"""Worker of tests/test_mmgcf_contract.py (own process: the kernels behind `mmrec_b200.ops` are patched).

MMGCF (`mmrec_b200.models.mmgcf`) under the harness of tests/dropin_contract_worker.py -- built the way quick_start builds
it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by
`install_cpu_ops`'s CPU stand-ins plus one for `ops.late_fuse`, the reference's torch expression on the gathered rows
(mmgcf_golden.torch_late_fuse), against tests/golden/mmgcf_tiny.npz and traj_mmgcf_*_tiny.npz recorded from the
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

import dualgnn_golden as G  # noqa: E402
import mmgcf_golden as M  # noqa: E402
import selfcf_golden  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402


def _data(text_only):
    from mmrec_b200.utils import synth
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, *rest = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, None if text_only else v, t)
    return rest


def _build(rest, over, epochs=None):
    Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = rest
    config = Config("MMGCF", "tiny", dict({"gpu_id": 0, "use_gpu": False}, **over, **extra))
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
    from mmrec_b200.models.mmgcf import MMGCF
    model = MMGCF(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def _install():
    install_cpu_ops()
    from mmrec_b200 import ops
    ops.late_fuse = M.torch_late_fuse


def _sub(gold, p):
    return {k[len(p):]: gold[k] for k in gold.files if k.startswith(p)}


def check_case(rest, name, gold):
    fusion, weighting, layers, _ = M.CASES[name]
    sub = _sub(gold, name + ".")
    config, model, valid_data, test_data, Trainer = _build(rest, M.overrides(fusion, weighting, layers))
    init = {k[len("init_sha256."):]: str(v) for k, v in sub.items() if k.startswith("init_sha256.")}
    out = {"init_identical": selfcf_golden.init_digests(model) == init
           and [k for k, _ in model.named_parameters()] == [str(x) for x in sub["param_order"]]}
    torch.manual_seed(M.PRUNE_SEED)
    draw = model.pruner.sample
    keep = []

    def once(dropout):
        adj, k = draw(dropout)
        keep.append(k)
        return adj, k
    model.pruner.sample = once
    model.pre_epoch_processing()                                         # the reference's draw on the CPU generator
    del model.pruner.sample
    _, _, v = model.masked_adj.coo()
    out["keep_equal"] = bool(np.array_equal(keep[0].numpy(), gold["prune_keep_idx"]))
    out["masked_vals_equal"] = bool(np.array_equal(np.sort(v.numpy()), np.sort(gold["masked_adj_val"])))
    model.eval()
    with torch.no_grad():
        u, i = model.forward(model.norm_adj)
        _, im = model.forward(model.masked_adj)
    out["fwd_rel"] = max(G.rel(sub, "fwd_i", i.numpy()), G.rel(sub, "fwd_masked_i", im.numpy()),
                         G.rel(sub, "fwd_u", u.numpy()) if "fwd_u.sha256" in sub else 0.0)
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    loss.backward()
    named = dict(model.named_parameters())
    grads = [k[5:] for k in G.recorded(sub, "grad.")]
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0]),
                "grad_keys": sorted(k for k, q in named.items() if q.grad is not None) == grads,
                "grad_rel": max(M.grad_errors(sub, {k: named[k].grad.numpy() for k in grads}).values())})
    model.zero_grad()
    model.eval()
    eb = [torch.from_numpy(gold["eval_users"]), torch.from_numpy(gold["eval_mask"])]
    with torch.no_grad():
        out["score_rel"] = G.rel(sub, "scores", model.full_sort_predict(eb).numpy())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in sub["metric_names"]]
    out["metric_max_abs"] = max(max(abs(valid[k] - w) for k, w in zip(names, sub["metric_values"])),
                                max(abs(test[k] - w) for k, w in zip(names, sub["test_metric_values"])))
    return out


def main_model():
    gold = np.load(os.path.join(HERE, "golden", "mmgcf_tiny.npz"), allow_pickle=True)
    _install()
    res = {}
    for text_only in (False, True):
        rest = _data(text_only)
        for name, case in M.CASES.items():
            if case[3] == text_only:
                res[name] = check_case(rest, name, gold)
    print("CONTRACT " + json.dumps(res))


def main_traj(name):
    gold = np.load(os.path.join(HERE, "golden", f"traj_mmgcf_{name}_tiny.npz"), allow_pickle=True)
    _install()
    rest = _data(False)
    fusion, weighting = M.TRAJ[name]
    config, model, valid_data, test_data, Trainer = _build(rest, M.overrides(fusion, weighting, 2, float(gold["dropout"])), epochs=2)
    trainer = Trainer(config, model)
    rec = {"losses": [], "valid": [], "test": [], "keep_equal": []}
    orig = model.calculate_loss

    def spy(interaction):
        l = orig(interaction)
        rec["losses"].append(float(l.detach()))
        return l
    model.calculate_loss = spy
    draw = model.pruner.sample

    def spy_sample(dropout):
        adj, keep = draw(dropout)
        rec["keep_equal"].append(bool(np.array_equal(keep.numpy(), gold["keep_idx"][len(rec["keep_equal"])])))
        return adj, keep
    model.pruner.sample = spy_sample
    offs = np.concatenate([[0], np.cumsum(gold["batch_sizes"])])
    first = np.concatenate([[0], np.cumsum(gold["batches_per_epoch"])])
    recorded = [[torch.from_numpy(gold["batches"][:, offs[b]:offs[b + 1]].copy()) for b in range(first[ep], first[ep + 1])]
                for ep in range(len(gold["batches_per_epoch"]))]
    for ep in range(2):
        torch.manual_seed(int(gold["seed0"]) + ep)
        model.pre_epoch_processing()
        trainer._train_epoch(recorded[ep], ep)
        trainer.lr_scheduler.step()
        rec["valid"].append(list(trainer.evaluate(valid_data).values()))
        rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    out = {"n_batches": len(rec["losses"]), "want_batches": int(gold["n_steps"]), "keep_equal": rec["keep_equal"],
           "loss_max_rel": float(np.max(np.abs(np.array(rec["losses"]) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(rec["valid"]) - gold["valid"]).max(), np.abs(np.array(rec["test"]) - gold["test"]).max()))}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    main_traj(arg[5:]) if arg.startswith("traj:") else main_model()
