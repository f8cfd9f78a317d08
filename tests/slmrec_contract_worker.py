"""Worker of tests/test_slmrec_contract.py: SLMRec (`mmrec_b200.models.slmrec`) under the harness of tests/contract.py,
with `install_cpu_ops`'s CPU stand-ins (`ops.project` = `F.linear`, `ops.propagate_mean` = `torch.sparse.mm` + stack + mean
on the [N, 3d] ego table, `ops.score` = the dense product), against tests/golden/slmrec_tiny.npz / traj_slmrec_tiny.npz
recorded from the reference's class."""
import sys

import numpy as np
import torch

import contract as C
import golden_io as G


def main_model():
    h = C.build("SLMRec")
    model, gold = h.model, C.case(C.load("slmrec_tiny.npz"))
    out = {"init_identical": C.check_init(model, gold)}
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(gold["batch"]))
    out["views_equal"] = {n: bool(np.array_equal(getattr(model, n).detach().numpy(), gold["view_" + n])) for n in ("i_emb", "v_emb", "t_emb")}
    out["tables_equal"] = bool(np.array_equal(model.all_users.detach().numpy(), gold["all_users"])
                               and np.array_equal(model.all_items.detach().numpy(), gold["all_items"]))
    loss.backward()
    named = dict(model.named_parameters())
    grads = {k[5:]: gold[k] for k in gold if k.startswith("grad.")}
    out.update({"loss": float(loss.item()), "want_loss": float(gold["loss"][0]),
                "grad_keys": sorted(k for k, p in named.items() if p.grad is not None) == sorted(grads),
                "grad_rel": {k: G.rel_to(named[k].grad.numpy(), g) for k, g in grads.items()},
                "grad_equal": sorted(k for k, g in grads.items() if np.array_equal(named[k].grad.numpy(), g))})
    model.zero_grad()
    sc = C.predict(model, gold)
    out["score_equal"] = bool(np.array_equal(sc, gold["scores"]))
    out["score_err"] = float(np.abs(sc - gold["scores"]).max())
    out.update(C.check_metrics(h, gold))
    C.emit(out)


def main_traj():
    h = C.build("SLMRec", after={"epochs": 2})
    C.emit(C.replay_trajectory(h, C.load("traj_slmrec_tiny.npz")))


if __name__ == "__main__":
    {"traj": main_traj}.get(sys.argv[1] if len(sys.argv) > 1 else "", main_model)()
