"""Worker of tests/test_mmgcf_contract.py: MMGCF (`mmrec_b200.models.mmgcf`) under the harness of tests/contract.py, with
`install_cpu_ops`'s CPU stand-ins plus one for `ops.late_fuse`, the reference's torch expression on the gathered rows
(mmgcf_golden.torch_late_fuse), against tests/golden/mmgcf_tiny.npz and traj_mmgcf_*_tiny.npz recorded from the
reference's class."""
import sys

import numpy as np
import torch

import contract as C
import golden_io as G
import mmgcf_golden as M


def install():
    from mmrec_b200 import ops
    ops.late_fuse = M.torch_late_fuse


def check_case(name, gold):
    fusion, weighting, layers, text_only = M.CASES[name]
    h = C.build("MMGCF", "t" if text_only else "vt", over=M.overrides(fusion, weighting, layers), batches={}, install=install)
    model, sub = h.model, C.case(gold, name + ".")
    out = {"init_identical": C.check_init(model, sub)}
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
    out["score_rel"] = G.rel(sub, "scores", C.predict(model, gold))
    out.update(C.check_metrics(h, sub))
    return out


def main_model():
    gold = C.load("mmgcf_tiny.npz")
    C.emit({name: check_case(name, gold) for text_only in (False, True) for name, case in M.CASES.items() if case[3] == text_only})


def main_traj(name):
    gold = C.load(f"traj_mmgcf_{name}_tiny.npz")
    fusion, weighting = M.TRAJ[name]
    h = C.build("MMGCF", over=M.overrides(fusion, weighting, 2, float(gold["dropout"])), batches={}, after={"epochs": 2},
                install=install)
    keep_equal = []
    draw = h.model.pruner.sample

    def spy_sample(dropout):
        adj, keep = draw(dropout)
        keep_equal.append(bool(np.array_equal(keep.numpy(), gold["keep_idx"][len(keep_equal)])))
        return adj, keep
    h.model.pruner.sample = spy_sample
    out = C.replay_trajectory(h, gold, lambda ep: torch.manual_seed(int(gold["seed0"]) + ep))
    out["keep_equal"] = keep_equal
    C.emit(out)


if __name__ == "__main__":
    arg = sys.argv[1] if len(sys.argv) > 1 else ""
    main_traj(arg[5:]) if arg.startswith("traj:") else main_model()
