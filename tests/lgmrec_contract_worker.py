"""Worker of tests/test_lgmrec_host.py: LGMRec (`mmrec_b200.models.lgmrec`) under the harness of tests/contract.py, with
the kernels replaced by CPU stand-ins, against tests/golden/lgmrec_*.npz recorded from the reference's class.  Every phase
runs under the torch seed make_golden_lgmrec.py set for it, so the class must draw the reference's Gumbel noise and dropout
masks itself; the draws are compared too.  The trajectory replays the recorded batches and draws."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

import contract as C
import golden_io as G
import lgmrec_golden

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


def install():
    from mmrec_b200 import ops
    ops.expsum_rows = expsum_rows


def _draws(gold, prefix):
    """The trajectory's recorded draws, in order."""
    return [gold["%sdraw%d" % (prefix, k)] for k in range(int(gold[prefix + "n_draws"]))]


def _same_draws(got, want):
    return len(got) == len(want) and all(a.shape == b.shape and np.array_equal(a, b) for a, b in zip(got, want))


def main_model(gfile):
    h = C.build("LGMRec", over=SETTINGS[gfile], install=install)
    model, gold = h.model, lgmrec_golden.load(os.path.join(C.GOLDEN, gfile))
    sd = model.state_dict()
    init_identical = all(np.array_equal(sd[k[len("param0."):]].numpy(), gold[k]) for k in gold.files if k.startswith("param0.")) \
        and [k for k, _ in model.named_parameters()] == [str(x) for x in gold["param_order"]]
    graphs = bool(np.array_equal(model.num_inters.numpy(), gold["num_inters"]))
    draws_ok = True
    model.eval()
    torch.manual_seed(SEEDS["fwd"])
    with Spy() as s, torch.no_grad():
        fu, fi, hyp = model.forward()
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "fwd_"))
    fwd_rel = max([G.rel_to(fu.numpy(), gold["fwd_u"]), G.rel_to(fi.numpy(), gold["fwd_i"])] +
                  [G.rel_to(x.numpy(), gold["fwd_hyper_" + n]) for n, x in zip(("uv", "iv", "ut", "it"), hyp)])
    model.train()
    torch.manual_seed(SEEDS["loss"])
    model.zero_grad()
    with Spy() as s:
        loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "loss_"))
    loss.backward()
    named = dict(model.named_parameters())
    grad_rel = max(G.rel_to(named[k[5:]].grad.numpy(), gold[k]) for k in gold.files if k.startswith("grad."))
    torch.manual_seed(SEEDS["scores"])
    with Spy() as s:
        sc = C.predict(model, gold)
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "scores_"))
    score_err = float(np.abs(sc - gold["scores"]).max() / np.abs(gold["scores"]).max())
    trainer = h.Trainer(h.config, model)
    torch.manual_seed(SEEDS["valid"])
    with Spy() as s:
        valid = trainer.evaluate(h.valid_data)
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "valid_"))
    torch.manual_seed(SEEDS["test"])
    with Spy() as s:
        test = trainer.evaluate(h.test_data, is_test=True)
    draws_ok &= _same_draws(s.draws, lgmrec_golden.regenerate(gold, "test_"))
    names = [str(x) for x in gold["metric_names"]]
    out = {"init_identical": bool(init_identical), "graphs": graphs, "draws_ok": bool(draws_ok), "fwd_rel": fwd_rel,
           "loss": float(loss.item()), "want_loss": float(gold["loss"][0]), "grad_rel": grad_rel, "score_err": score_err,
           "valid": {k: float(v) for k, v in valid.items()}, "want_valid": dict(zip(names, [float(x) for x in gold["metric_values"]])),
           "test": {k: float(v) for k, v in test.items()}, "want_test": dict(zip(names, [float(x) for x in gold["test_metric_values"]]))}
    C.emit(out)


def main_traj():
    h = C.build("LGMRec", after={"epochs": 2}, install=install)
    gold = C.load("traj_lgmrec_tiny.npz")
    with Spy(replay=_draws(gold, "")) as s:
        out = C.replay_trajectory(h, gold)
    out["draws_left"] = len(s.replay)
    C.emit(out)


if __name__ == "__main__":
    arg = sys.argv[1]
    main_traj() if arg == "traj" else main_model(arg)
