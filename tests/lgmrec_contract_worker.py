"""Worker of tests/test_lgmrec_host.py (own process: the kernels behind `mmrec_b200.ops` are patched).

LGMRec (`mmrec_b200.models.lgmrec`) under the harness of tests/dropin_contract_worker.py -- built the way quick_start builds
it, the package's restatement or, with MMREC_REFERENCE_SRC, the reference's own code -- with the kernels replaced by CPU
stand-ins, against tests/golden/lgmrec_*.npz recorded from the reference's class.  Every phase runs under the torch seed
make_golden_lgmrec.py set for it, so the class must draw the reference's Gumbel noise and dropout masks itself; the draws are
compared too.  The trajectory replays the recorded batches and draws."""
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

import lgmrec_golden  # noqa: E402
from dropin_contract_worker import harness, install_cpu_ops  # noqa: E402

SEEDS = {"fwd": 11, "loss": 4321, "scores": 12, "valid": 13, "test": 14}      # as tests/golden/make_golden_lgmrec.py
SETTINGS = {"lgmrec_tiny.npz": {},
            "lgmrec_clothing_tiny.npz": {"n_hyper_layer": [2], "hyper_num": [64], "keep_rate": [0.2], "alpha": [0.2]}}
_gumbel, _dropout = F.gumbel_softmax, F.dropout


class Spy:
    """`F.gumbel_softmax` / `F.dropout` restated as make_golden_lgmrec.py restates them (it proves the restatement
    bit-identical to torch's own functions): draws from torch's generator and records the draws, or (`replay`) takes the
    recorded ones in order."""

    def __init__(self, replay=None):
        self.draws, self.replay = [], None if replay is None else list(replay)

    def gumbel_softmax(self, logits, tau=1.0, hard=False, eps=1e-10, dim=-1):
        g = torch.from_numpy(self.replay.pop(0)) if self.replay is not None else \
            -torch.empty_like(logits, memory_format=torch.legacy_contiguous_format).exponential_().log()
        self.draws.append(g.numpy().copy())
        return ((logits + g) / tau).softmax(dim)

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

    def __enter__(self):
        F.gumbel_softmax, F.dropout = self.gumbel_softmax, self.dropout
        return self

    def __exit__(self, *exc):
        F.gumbel_softmax, F.dropout = _gumbel, _dropout


def expsum_rows(q, t, tau):                                           # the stand-in restates lgmrec.py:164
    return torch.exp(torch.matmul(q, t.T) / tau).sum(dim=1)


def _setup(over, epochs=None):
    from mmrec_b200.utils import synth
    torch.set_num_threads(1)
    tmp = tempfile.mkdtemp(prefix="mmrec_contract_")
    data, Config, RecDataset, TrainDataLoader, EvalDataLoader, init_seed, Trainer, extra = harness(tmp)
    u, i, e, d, f = synth.SHAPES["tiny"]
    g = synth.make_graph(u, i, e, seed=0)
    v, t = synth.make_features(i, f, seed=1)
    synth.write_dataset(data, "tiny", g, v, t)
    config = Config("LGMRec", "tiny", dict({"gpu_id": 0, "use_gpu": False, "eval_batch_size": 128, "train_batch_size": 512}, **over, **extra))
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
    ops.expsum_rows = expsum_rows
    from mmrec_b200.models.lgmrec import LGMRec
    model = LGMRec(config, train_data).to(config["device"])
    return config, model, valid_data, test_data, Trainer


def _draws(gold, prefix):
    """The trajectory's recorded draws, in order."""
    return [gold["%sdraw%d" % (prefix, k)] for k in range(int(gold[prefix + "n_draws"]))]


def _same_draws(got, want):
    return len(got) == len(want) and all(a.shape == b.shape and np.array_equal(a, b) for a, b in zip(got, want))


def main_model(gfile):
    config, model, valid_data, test_data, Trainer = _setup(SETTINGS[gfile])
    gold = lgmrec_golden.load(os.path.join(HERE, "golden", gfile))
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0.")) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    graphs = bool(np.array_equal(model.num_inters.numpy(), gold["num_inters"]))

    def rel(a, b):
        return float(np.linalg.norm(np.asarray(a, dtype=np.float64) - b) / max(np.linalg.norm(b), 1e-30))
    draws_ok = True
    model.eval()
    torch.manual_seed(SEEDS["fwd"])
    with Spy() as s, torch.no_grad():
        fu, fi, hyp = model.forward()
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "fwd_"))
    fwd_rel = max([rel(fu.numpy(), gold["fwd_u"]), rel(fi.numpy(), gold["fwd_i"])] +
                  [rel(h.numpy(), gold["fwd_hyper_" + n]) for n, h in zip(("uv", "iv", "ut", "it"), hyp)])
    model.train()
    torch.manual_seed(SEEDS["loss"])
    model.zero_grad()
    with Spy() as s:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "loss_"))
    loss.backward()
    named = dict(model.named_parameters())
    grad_rel = max(rel(named[k[5:]].grad.numpy(), gold[k]) for k in gold.files if k.startswith("grad."))
    model.eval()
    torch.manual_seed(SEEDS["scores"])
    with Spy() as s, torch.no_grad():
        sc = model.full_sort_predict([torch.from_numpy(gold["eval_users"]), torch.from_numpy(gold["eval_mask"])])
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "scores_"))
    score_err = float(np.abs(sc.numpy() - gold["scores"]).max() / np.abs(gold["scores"]).max())
    trainer = Trainer(config, model)
    torch.manual_seed(SEEDS["valid"])
    with Spy() as s:
        valid = trainer.evaluate(valid_data)
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "valid_"))
    torch.manual_seed(SEEDS["test"])
    with Spy() as s:
        test = trainer.evaluate(test_data, is_test=True)
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "test_"))
    names = [str(x) for x in gold["metric_names"]]
    out = {"init_identical": bool(init_identical), "graphs": graphs, "draws_ok": bool(draws_ok), "fwd_rel": fwd_rel,
           "loss": float(loss.item()), "want_loss": float(gold["loss"][0]), "grad_rel": grad_rel, "score_err": score_err,
           "valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in gold["metric_values"]])),
           "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in gold["test_metric_values"]]))}
    print("CONTRACT " + json.dumps(out))


def main_traj():
    config, model, valid_data, test_data, Trainer = _setup({}, epochs=2)
    gold = np.load(os.path.join(HERE, "golden", "traj_lgmrec_tiny.npz"), allow_pickle=True)
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
    with Spy(replay=_draws(gold, "")) as s:
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
    arg = sys.argv[1]
    main_traj() if arg == "traj" else main_model(arg)
