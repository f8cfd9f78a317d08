"""Worker of tests/test_mvgae_host.py: MVGAE (`mmrec_b200.models.mvgae`) under the harness of tests/contract.py, with the
kernels replaced by CPU stand-ins, against tests/golden/mvgae_tiny.npz / traj_mvgae_tiny.npz recorded from the reference's
class.  The loss phase runs under the torch seed make_golden_mvgae.py set for it, so the class must draw the reference's
dropout masks and Gaussian noise itself; the draws are compared too.  The trajectory replays the recorded batches and draws.

The stand-in for `ops.max_dot` evaluates the scores in float64: the recorded argmax (the reference's fp32 sum) is required
except at near ties, where the two candidates' float64 scores are within the fp32 error bound of the reference's sum."""
import sys

import numpy as np
import torch
import torch.nn.functional as F

import contract as C
import golden_io as G
import mvgae_golden

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


def install():
    from mmrec_b200 import ops
    ops.max_dot = max_dot


def main_model():
    h = C.build("MVGAE", install=install)
    model, gold = h.model, C.case(C.load("mvgae_tiny.npz"))
    init_identical = C.check_init(model, gold, mvgae_golden.plain(model))
    draws_ok = True
    model.eval()
    with Spy() as s, torch.no_grad():
        fwd = model.forward()
    draws_ok &= not s.draws
    fwd_rel = max(G.rel_to(fwd[0].numpy(), gold["fwd_pd_mu"]), G.rel_to(fwd[2].numpy(), gold["fwd_pd_mu"]))
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
        dec_rel = max(dec_rel, G.rel_to(v.numpy(), gold["decode_val"][c]))
        want_i = torch.from_numpy(gold["decode_arg"][c])
        for b in torch.nonzero(i != want_i).flatten().tolist():
            n_diff += 1
            gap = float(sc[b, i[b]] - sc[b, want_i[b]])
            tie_ok &= gap <= 2 * gamma * float(bound[b]) + 1e-6 * float(v[b].abs())
    named = dict(model.named_parameters())
    grad_keys = sorted(k for k, p in named.items() if p.grad is not None) == sorted(k[5:] for k in gold if k.startswith("grad."))
    grad_rel = max(G.rel_to(named[k[5:]].grad.numpy(), gold[k]) for k in gold if k.startswith("grad."))
    sc = C.predict(model, gold)
    score_err = float(np.abs(sc - gold["scores"]).max() / np.abs(gold["scores"]).max())
    out = {"init_identical": bool(init_identical), "draws_ok": bool(draws_ok), "fwd_rel": fwd_rel, "n_decodes": len(DECODES),
           "decode_rel": dec_rel, "argmax_diff": n_diff, "argmax_near_ties": bool(tie_ok),
           "loss": float(loss.item()), "want_loss": float(gold["loss"][0]), "grad_keys": bool(grad_keys), "grad_rel": grad_rel,
           "score_err": score_err}
    out.update(C.check_metrics(h, gold))
    C.emit(out)


def main_traj():
    h = C.build("MVGAE", after={"epochs": 2}, install=install)
    gold = C.load("traj_mvgae_tiny.npz")
    with Spy(replay=mvgae_golden.trajectory_draws(gold)) as s:
        out = C.replay_trajectory(h, gold)
    out["draws_left"] = len(s.replay)
    C.emit(out)


if __name__ == "__main__":
    main_traj() if sys.argv[1] == "traj" else main_model()
