"""Worker of tests/test_selfcf_host.py (own process: the kernels behind `mmrec_b200.ops` are patched).

SELFCFED_LGN (`mmrec_b200.models.selfcfed_lgn`, with its encoder `mmrec_b200.common.encoders.LightGCN_Encoder`) under the
harness of tests/dropin_contract_worker.py -- built the way quick_start builds it, the package's restatement or, with
MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by CPU stand-ins, against
tests/golden/selfcfed_lgn_tiny.npz / traj_selfcfed_lgn_tiny.npz recorded from the reference's class.

On the CPU the class draws everything itself from the seeded generators, as the reference did: the rate
(`np.random.random()`), `torch.rand(nnz)` and the two target masks; `selfcf_golden.Replay` seeds each phase and records the
draws' digests, which must equal the recorded ones.  The stand-ins:
- `ops.edge_keep_bits`: the keep rule `floor(float32(1 - rate) + r) != 0` as a bool mask in CSR order through `draw_of`
  (and its mirror through `mirror`), in place of the packed bits;
- `ops.propagate_mean_dropped`: the oracle restatement of `sparse_dropout` + `torch.sparse.mm` (encoders.py:77-112): the
  kept entries of the CPU CSR, values times float32(scale), `oracle.propagate_mean` under torch autograd;
- `ops.propagate_mean_fused`: `oracle.propagate_mean` of the undropped matrix;
- `ops.score`: `install_cpu_ops`'s dense product (of the width-2d operands)."""
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

MASKS = []


def install_selfcf_ops():
    from oracle import mmrec_oracle as O
    from mmrec_b200 import ops

    def edge_keep_bits(draws, keep_prob, draw_of, mirror=None):
        keep = torch.floor(draws[draw_of.long()] + np.float32(keep_prob)) != 0
        MASKS.append(keep)
        return keep, None if mirror is None else keep[mirror.long()]

    def propagate_mean_dropped(A, ego, n_layers, keep, keep_t, scale):
        assert A.symmetric
        r, c, v = A.coo()
        dropped = torch.sparse_coo_tensor(torch.stack((r[keep], c[keep])), v[keep] * np.float32(scale), (A.n_rows, A.n_cols))
        return O.propagate_mean(dropped, ego, n_layers)

    def propagate_mean_fused(A, ego, n_layers, cooperative=True, **kw):
        assert not kw
        return O.propagate_mean(A.t_, torch.cat(ego) if isinstance(ego, (tuple, list)) else ego, n_layers)

    ops.edge_keep_bits = edge_keep_bits
    ops.propagate_mean_dropped = propagate_mean_dropped
    ops.propagate_mean_fused = propagate_mean_fused


def _setup(epochs=None, n_layers=None):
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    over = {"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}
    if n_layers is not None:
        over["n_layers"] = n_layers
    config = Config("SELFCFED_LGN", "tiny", dict(over, **extra))
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
    install_selfcf_ops()
    from mmrec_b200.models.selfcfed_lgn import SELFCFED_LGN
    model = SELFCFED_LGN(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / max(np.linalg.norm(b), 1e-30))


def loss_phase(model, gold, prefix):
    """One seeded `calculate_loss` + backward on the recorded batch against the fields under `prefix`."""
    model.train()
    model.zero_grad()
    fwd = []
    orig = model.forward

    def spy(inputs):
        o = orig(inputs)
        fwd.append((o[0].detach(), o[2].detach()))
        return o
    model.forward = spy
    MASKS.clear()
    with selfcf_golden.Replay(gold[prefix + "loss_seed"]) as rep:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    del model.forward
    loss.backward()
    named = dict(model.named_parameters())
    grads = {k[len(prefix) + 5:]: gold[k] for k in gold.files if k.startswith(prefix + "grad.")}
    out = {"draws_ok": rep.digests == [str(x) for x in gold[prefix + "loss_draw_sha256"]] and len(MASKS) == 1,
           "n_kept": int(MASKS[0].sum()) if MASKS else -1, "nnz": int(MASKS[0].numel()) if MASKS else -1,
           "fwd_u_equal": bool(np.array_equal(fwd[0][0].numpy(), gold[prefix + "fwd_u_online"])),
           "fwd_i_equal": bool(np.array_equal(fwd[0][1].numpy(), gold[prefix + "fwd_i_online"])),
           "loss": float(loss.item()), "want_loss": float(gold[prefix + "loss"][0]),
           "grad_keys": sorted(k for k, p in named.items() if p.grad is not None) == sorted(grads),
           "grad_rel": max(rel(named[k].grad.numpy(), g) for k, g in grads.items())}
    model.zero_grad()
    return out


def main_model():
    config, model, valid_data, test_data, Trainer = _setup()
    gold = np.load(os.path.join(HERE, "golden", "selfcfed_lgn_tiny.npz"), allow_pickle=True)
    init_identical = not selfcf_golden.same_init(model, gold) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    out = {"init_identical": bool(init_identical), "n_layers": model.online_encoder.n_layers}
    out.update(loss_phase(model, gold, ""))
    model.eval()
    with torch.no_grad():
        sc = model.full_sort_predict([torch.from_numpy(gold["eval_users"]), torch.from_numpy(gold["eval_mask"])])
    out["score_err"] = float(np.abs(sc.numpy() - gold["scores"]).max() / np.abs(gold["scores"]).max())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in gold["metric_names"]]
    out.update({"valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in gold["metric_values"]])),
                "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in gold["test_metric_values"]]))})
    print("CONTRACT " + json.dumps(out))


def main_two_layers():
    config, model, _, _, _ = _setup(n_layers=2)
    gold = np.load(os.path.join(HERE, "golden", "selfcfed_lgn_tiny.npz"), allow_pickle=True)
    out = {"init_identical": not selfcf_golden.same_init(model, gold), "n_layers": model.online_encoder.n_layers}
    out.update(loss_phase(model, gold, "l2_"))
    print("CONTRACT " + json.dumps(out))


def main_traj():
    config, model, valid_data, test_data, Trainer = _setup(epochs=2)
    gold = np.load(os.path.join(HERE, "golden", "traj_selfcfed_lgn_tiny.npz"), allow_pickle=True)
    trainer = Trainer(config, model)
    rec = {"losses": [], "valid": [], "test": [], "draws_ok": True}
    orig = model.calculate_loss

    def spy(interaction):
        b = len(rec["losses"])
        with selfcf_golden.Replay(int(gold["seed0"]) + b) as rep:
            l = orig(interaction)
        rec["draws_ok"] &= rep.digests == [str(x) for x in gold["draw_sha256"][b]]
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
    out = {"n_batches": len(rec["losses"]), "want_batches": int(gold["n_steps"]), "draws_ok": bool(rec["draws_ok"]),
           "loss_max_rel": float(np.max(np.abs(np.array(rec["losses"]) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(rec["valid"]) - gold["valid"]).max(), np.abs(np.array(rec["test"]) - gold["test"]).max()))}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    {"traj": main_traj, "layers2": main_two_layers}.get(sys.argv[1], main_model)()
