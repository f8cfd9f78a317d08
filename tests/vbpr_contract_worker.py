"""Worker of tests/test_vbpr_contract.py: VBPR and BPR (`mmrec_b200.models.vbpr`, `.bpr`) under the harness of
tests/contract.py, with `install_cpu_ops`'s CPU stand-ins plus one for `ops.bpr_mf_loss`, the reference's torch expression on
the gathered rows (vbpr_golden.torch_bpr_mf_loss), against tests/golden/{vbpr,bpr}_tiny.npz and traj_{vbpr,bpr}_tiny.npz
recorded from the reference's classes."""
import sys

import numpy as np
import torch

import contract as C
import golden_io as G
import vbpr_golden as V


def install():
    from mmrec_b200 import ops
    ops.bpr_mf_loss = V.torch_bpr_mf_loss


def main_model(p):
    name, mods = V.CASES[p]
    h = C.build(name, mods, install=install)
    model, sub = h.model, C.case(C.load(f"{name.lower()}_tiny.npz"), p)
    out = {"init_identical": C.check_init(model, sub)}
    model.train()
    model.zero_grad()
    loss = model.calculate_loss(torch.from_numpy(sub["batch"]))
    loss.backward()
    out["grad_keys"], out["grad_rel"] = C.check_grads(model, sub)
    out.update({"loss": float(loss.item()), "want_loss": float(sub["loss"][0]), "loss_shape": list(loss.shape)})
    model.zero_grad()
    out["score_rel"] = G.rel(sub, "scores", C.predict(model, sub))
    out.update(C.check_metrics(h, sub))
    C.emit(out)


def main_traj(name):
    h = C.build(name, V.TRAJ[name], after={"epochs": 2}, install=install)
    gold = C.load(f"traj_{name.lower()}_tiny.npz")
    rng_kept = []
    orig = h.model.calculate_loss

    def spy(interaction):
        st = torch.get_rng_state()
        l = orig(interaction)
        rng_kept.append(bool(torch.equal(st, torch.get_rng_state())))
        return l
    h.model.calculate_loss = spy
    out = C.replay_trajectory(h, gold)
    out["rng_kept"] = all(rng_kept) and bool(np.all(gold["rng_kept"]))
    C.emit(out)


if __name__ == "__main__":
    arg = sys.argv[1]
    main_traj(arg[5:]) if arg.startswith("traj:") else main_model(arg)
