"""Worker of tests/test_mvgae_host.py (own process: the kernels behind `mmrec_b200.ops` are patched).

MVGAE (`mmrec_b200.models.mvgae`) under the harness of tests/dropin_contract_worker.py -- built the way quick_start builds
it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by CPU
stand-ins, against tests/golden/mvgae_tiny.npz / traj_mvgae_tiny.npz recorded from the reference's class.  The loss phase
runs under the torch seed make_golden_mvgae.py set for it, so the class must draw the reference's dropout masks and
Gaussian noise itself; the draws are compared too.  The trajectory replays the recorded batches and draws.

The stand-in for `ops.max_dot` evaluates the scores in float64: the recorded argmax (the reference's fp32 sum) is required
except at near ties, where the two candidates' float64 scores are within the fp32 error bound of the reference's sum."""
import json
import os
import sys
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, HERE)

import mvgae_golden  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402

SEEDS = {"loss": 4321}                                                # as tests/golden/make_golden_mvgae.py
_dropout, _randn_like = F.dropout, torch.randn_like


class Spy:
    """`F.dropout` / `torch.randn_like` restated as make_golden_mvgae.py restates them (it proves the restatement
    bit-identical to torch's own functions): draws from torch's generator and records the draws, or (`replay`) takes the
    recorded ones in order."""

    def __init__(self, replay=None):
        self.draws, self.replay = [], None if replay is None else list(replay)

    def dropout(self, input, p=0.5, training=True, inplace=False):
        if not training or p == 0 or input.numel() == 0:
            return input
        if self.replay is not None:
            noise = torch.from_numpy(self.replay.pop(0))
        else:
            noise = torch.empty_like(input).bernoulli_(1 - p)
            noise.div_(1 - p)
        self.draws.append(noise.numpy().copy())
        return input * noise

    def randn_like(self, input, **kw):
        x = torch.from_numpy(self.replay.pop(0)) if self.replay is not None else torch.empty_like(input).normal_()
        self.draws.append(x.numpy().copy())
        return x

    def __enter__(self):
        F.dropout, torch.randn_like = self.dropout, self.randn_like
        return self

    def __exit__(self, *exc):
        F.dropout, torch.randn_like = _dropout, _randn_like


DECODES = []


def max_dot(q, t):
    """Stand-in for ops.max_dot: the max over j of <q_b, t_j> in float64 (first index on ties), differentiable in values."""
    s = q.double() @ t.double().T
    v, i = torch.max(s, dim=-1)
    with torch.no_grad():
        bound = (q.double().abs() @ t.double().abs().T).gather(1, i.unsqueeze(1)).squeeze(1)     # sum_k |q_k t_k| at the max
    DECODES.append((s.detach(), v.detach(), i, bound))
    return v.float(), i


def _setup(epochs=None):
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    config = Config("MVGAE", "tiny", dict({"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}, **extra))
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
    ops.max_dot = max_dot
    from mmrec_b200.models.mvgae import MVGAE
    model = MVGAE(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / max(np.linalg.norm(b), 1e-30))


def main_model():
    config, model, valid_data, test_data, Trainer = _setup()
    gold = np.load(os.path.join(HERE, "golden", "mvgae_tiny.npz"), allow_pickle=True)
    init_identical = not mvgae_golden.same_init(model, gold) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    draws_ok = True
    model.eval()
    with Spy() as s, torch.no_grad():
        fwd = model.forward()
    draws_ok &= not s.draws
    fwd_rel = max(rel(fwd[0].numpy(), gold["fwd_pd_mu"]), rel(fwd[2].numpy(), gold["fwd_pd_mu"]))
    model.train()
    torch.manual_seed(SEEDS["loss"])
    model.zero_grad()
    DECODES.clear()
    with Spy() as s:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    want = mvgae_golden.regenerate(gold, "loss_")
    draws_ok &= len(s.draws) == len(want) and all(np.array_equal(a, b) for a, b in zip(s.draws, want))
    loss.backward()
    # the decode: values, and the recorded argmax except at near ties (float64 gap within the fp32 bound gamma_d sum|q_k t_k|)
    d = model.dim_x
    gamma = d * 2.0 ** -24 / (1 - d * 2.0 ** -24)
    dec_rel, n_diff, tie_ok = 0.0, 0, True
    for c, (sc, v, i, bound) in enumerate(DECODES):
        dec_rel = max(dec_rel, rel(v.numpy(), gold["decode_val"][c]))
        want_i = torch.from_numpy(gold["decode_arg"][c])
        for b in torch.nonzero(i != want_i).flatten().tolist():
            n_diff += 1
            gap = float(sc[b, i[b]] - sc[b, want_i[b]])
            tie_ok &= gap <= 2 * gamma * float(bound[b]) + 1e-6 * float(v[b].abs())
    named = dict(model.named_parameters())
    grad_keys = sorted(k for k, p in named.items() if p.grad is not None) == sorted(k[5:] for k in gold.files if k.startswith("grad."))
    grad_rel = max(rel(named[k[5:]].grad.numpy(), gold[k]) for k in gold.files if k.startswith("grad."))
    model.eval()
    with torch.no_grad():
        sc = model.full_sort_predict([torch.from_numpy(gold["eval_users"]), torch.from_numpy(gold["eval_mask"])])
    score_err = float(np.abs(sc.numpy() - gold["scores"]).max() / np.abs(gold["scores"]).max())
    trainer = Trainer(config, model)
    valid = trainer.evaluate(valid_data)
    test = trainer.evaluate(test_data, is_test=True)
    names = [str(x) for x in gold["metric_names"]]
    out = {"init_identical": bool(init_identical), "draws_ok": bool(draws_ok), "fwd_rel": fwd_rel, "n_decodes": len(DECODES),
           "decode_rel": dec_rel, "argmax_diff": n_diff, "argmax_near_ties": bool(tie_ok),
           "loss": float(loss.item()), "want_loss": float(gold["loss"][0]), "grad_keys": bool(grad_keys), "grad_rel": grad_rel,
           "score_err": score_err,
           "valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in gold["metric_values"]])),
           "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in gold["test_metric_values"]]))}
    print("CONTRACT " + json.dumps(out))


def main_traj():
    config, model, valid_data, test_data, Trainer = _setup(epochs=2)
    gold = np.load(os.path.join(HERE, "golden", "traj_mvgae_tiny.npz"), allow_pickle=True)
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
    with Spy(replay=mvgae_golden.trajectory_draws(gold)) as s:
        for ep in range(2):
            model.pre_epoch_processing()
            trainer._train_epoch(recorded[ep], ep)
            trainer.lr_scheduler.step()
            rec["valid"].append(list(trainer.evaluate(valid_data).values()))
            rec["test"].append(list(trainer.evaluate(test_data, is_test=True).values()))
    out = {"n_batches": len(rec["losses"]), "draws_left": len(s.replay),
           "loss_max_rel": float(np.max(np.abs(np.array(rec["losses"]) - gold["losses"]) / np.abs(gold["losses"]))),
           "metric_max_abs": float(max(np.abs(np.array(rec["valid"]) - gold["valid"]).max(), np.abs(np.array(rec["test"]) - gold["test"]).max()))}
    print("CONTRACT " + json.dumps(out))


if __name__ == "__main__":
    main_traj() if sys.argv[1] == "traj" else main_model()
