"""Worker of tests/test_selfcf_contract.py: SELFCFED_LGN (`mmrec_b200.models.selfcfed_lgn`, with its encoder
`mmrec_b200.common.encoders.LightGCN_Encoder`) under the harness of tests/contract.py, with the kernels replaced by CPU
stand-ins, against tests/golden/selfcfed_lgn_tiny.npz / traj_selfcfed_lgn_tiny.npz recorded from the reference's class.

On the CPU the class draws everything itself from the seeded generators, as the reference did: the rate
(`np.random.random()`), `torch.rand(nnz)` and the two target masks; `selfcf_golden.Replay` seeds each phase and records the
draws' digests, which must equal the recorded ones.  The stand-ins:
- `ops.edge_keep_bits`: the keep rule `floor(float32(1 - rate) + r) != 0` as a bool mask in CSR order through `draw_of`
  (and its mirror through `mirror`), in place of the packed bits;
- `ops.propagate_mean_dropped`: the oracle restatement of `sparse_dropout` + `torch.sparse.mm` (encoders.py:77-112): the
  kept entries of the CPU CSR, values times float32(scale), `oracle.propagate_mean` under torch autograd;
- `ops.propagate_mean_fused`: `oracle.propagate_mean` of the undropped matrix;
- `ops.score`: `install_cpu_ops`'s dense product (of the width-2d operands)."""
import sys

import numpy as np
import torch

import contract as C
import golden_io as G
import selfcf_golden

MASKS = []


def install():
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
           "grad_rel": max(G.rel_to(named[k].grad.numpy(), g) for k, g in grads.items())}
    model.zero_grad()
    return out


def main_model():
    h = C.build("SELFCFED_LGN", install=install)
    model, gold = h.model, C.load("selfcfed_lgn_tiny.npz")
    out = {"init_identical": C.check_init(model, gold), "n_layers": model.online_encoder.n_layers}
    out.update(loss_phase(model, gold, ""))
    out["score_err"] = float(np.abs(C.predict(model, gold) - gold["scores"]).max() / np.abs(gold["scores"]).max())
    out.update(C.check_metrics(h, gold))
    C.emit(out)


def main_two_layers():
    model = C.build("SELFCFED_LGN", over={"n_layers": 2}, install=install).model
    gold = C.load("selfcfed_lgn_tiny.npz")
    out = {"init_identical": not G.same_init(model, gold), "n_layers": model.online_encoder.n_layers}
    out.update(loss_phase(model, gold, "l2_"))
    C.emit(out)


def main_traj():
    h = C.build("SELFCFED_LGN", after={"epochs": 2}, install=install)
    gold = C.load("traj_selfcfed_lgn_tiny.npz")
    draws_ok = []
    orig = h.model.calculate_loss

    def spy(interaction):
        b = len(draws_ok)
        with selfcf_golden.Replay(int(gold["seed0"]) + b) as rep:
            l = orig(interaction)
        draws_ok.append(rep.digests == [str(x) for x in gold["draw_sha256"][b]])
        return l
    h.model.calculate_loss = spy
    out = C.replay_trajectory(h, gold)
    out["draws_ok"] = all(draws_ok)
    C.emit(out)


if __name__ == "__main__":
    {"traj": main_traj, "layers2": main_two_layers}.get(sys.argv[1], main_model)()
