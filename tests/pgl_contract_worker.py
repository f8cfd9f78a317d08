"""Worker of tests/test_pgl_contract.py: PGL (`mmrec_b200.models.pgl`) under the harness of tests/contract.py, with
`install_cpu_ops`'s CPU stand-ins plus one for `ops.pgl_loss`, the reference's torch expression on the gathered rows with the
model's masks (pgl_golden.torch_pgl_loss), against tests/golden/pgl_tiny.npz and traj_pgl_tiny.npz recorded from the
reference's class."""
import sys

import numpy as np
import torch

import contract as C
import golden_io as G
import pgl_golden as P


def install():
    from mmrec_b200 import ops
    ops.pgl_loss = P.torch_pgl_loss


def spy_keep(model):
    """Record the keep indices of every `pre_epoch_processing` draw."""
    kept, orig = [], model.pruner.sample

    def sample(*a, **k):
        adj, keep = orig(*a, **k)
        kept.append(keep.numpy().copy())
        return adj, keep
    model.pruner.sample = sample
    return kept


def main_model():
    h = C.build("PGL", "vt", install=install)
    model, gold = h.model, C.load("pgl_tiny.npz")
    out = {"init_identical": C.check_init(model, gold)}
    kept = spy_keep(model)
    torch.manual_seed(P.PRUNE_SEED)
    model.pre_epoch_processing()
    out["same_keep"] = bool(np.array_equal(kept[0], gold["keep_idx"]))
    model.eval()
    with torch.no_grad():
        out["fwd_rel"] = max(G.rel(gold, f"{tag}_{s}", t.numpy()) for tag, adj in (("fwd_sub", model.sub_graph), ("fwd_norm", model.norm_adj))
                             for s, t in zip("ui", model.forward(adj)))
    drawn, orig = [], model._dropout_masks

    def masks(*a):
        m = orig(*a)
        drawn.append(torch.stack(m).numpy())
        return m
    model._dropout_masks = masks
    model.train()
    batch = torch.from_numpy(gold["batch"])
    out["cases"] = {}
    for p, rw in P.REG_CASES.items():
        sub = C.case(gold, p, tuple(P.REG_CASES))
        model.reg_weight = rw
        torch.manual_seed(P.LOSS_SEED)
        model.zero_grad(set_to_none=True)
        loss = model.calculate_loss(batch)
        loss.backward()
        r = {"same_masks": bool(np.array_equal(drawn[-1], P.masks_of(gold).numpy())), "loss": float(loss.item()),
             "want_loss": float(sub["loss"][0]), "loss_shape": list(loss.shape)}
        r["grad_keys"], r["grad_rel"] = C.check_grads(model, sub)
        out["cases"][p] = r
    model.zero_grad(set_to_none=True)
    out["score_rel"] = G.rel(gold, "scores", C.predict(model, gold))
    out.update(C.check_metrics(h, gold))
    C.emit(out)


def main_traj():
    h = C.build("PGL", "vt", over=dict(P.TRAJ_OVER), after={"epochs": 2}, install=install)
    gold = C.load("traj_pgl_tiny.npz")
    kept = spy_keep(h.model)
    out = C.replay_trajectory(h, gold, before_epoch=lambda ep: torch.manual_seed(P.TRAJ_SEED0 + ep))
    out["same_keep"] = len(kept) == 2 and all(np.array_equal(k, w) for k, w in zip(kept, gold["keep_idx"]))
    C.emit(out)


if __name__ == "__main__":
    main_traj() if sys.argv[1:] == ["traj"] else main_model()
