"""The random draws of MVGAE's golden files (tests/golden/mvgae_tiny.npz, traj_mvgae_tiny.npz; make_golden_mvgae.py).

A training forward of MVGAE draws nine `F.dropout` masks (three per GCN, in the order v, t, c; p = 0.1) and then four
`torch.randn_like` tensors (z, then z_v, z_t, z_c), all [n_users + n_items, embedding_size].  Per recorded phase the files
keep the torch seed and, per draw, its kind, shape, dropout probability and the SHA-256 of its fp32 bytes
(`lgmrec_golden.pack`).  The draws are regenerated here from a CPU `torch.Generator` with that seed: the reference drew them
from torch's default CPU generator seeded the same way at the start of the phase and consumed by nothing else within it,
which make_golden_mvgae.py asserts.  (The noise is incompressible fp32: 100 KiB per draw at `tiny`, 3 MiB over the
trajectory's eight batches.)"""
import numpy as np
import torch

from lgmrec_golden import digest, pack  # noqa: F401  (re-exported for the generator)


def regenerate(gold, prefix):
    """The draws of one phase as fp32 arrays, in order; each checked against its recorded digest."""
    gen = torch.Generator().manual_seed(int(gold[prefix + "seed"]))
    out = []
    for k in range(int(gold[prefix + "n_draws"])):
        kind, shape, p = str(gold[prefix + "draw_kind"][k]), tuple(int(x) for x in gold[prefix + "draw_shape"][k]), float(gold[prefix + "draw_p"][k])
        if kind == "randn":                                           # torch.randn_like: empty_like(x).normal_()
            x = torch.empty(shape).normal_(generator=gen)
        else:                                                         # F.dropout (CPU): empty_like(x).bernoulli_(1 - p).div_(1 - p)
            x = torch.empty(shape).bernoulli_(1 - p, generator=gen)
            x.div_(1 - p)
        a = x.numpy()
        assert digest(a) == str(gold[prefix + "draw_sha256"][k]), f"{prefix}draw {k}: torch's CPU generator no longer gives the recorded draw"
        out.append(a)
    return out


def init_digests(model) -> dict:
    """SHA-256 of the fp32 bytes of every initial state: the `state_dict` entries (`param0.<name>`) and the plain tensors the
    reference keeps beside its parameters (`plain.collaborative`, `plain.{v,t,c}_preference`, `plain.result_embed0`).  The
    file keeps these digests, not the 1.2 MiB of incompressible weights: equal digests are equal bits."""
    out = {"param0." + k: digest(v.detach().cpu().numpy()) for k, v in model.state_dict().items()}
    out["plain.collaborative"] = digest(model.collaborative.detach().cpu().numpy())
    for m in "vtc":
        out["plain.%s_preference" % m] = digest(getattr(model, m + "_gcn").preference.detach().cpu().numpy())
    out["plain.result_embed0"] = digest(model.result_embed.detach().cpu().numpy())
    return out


def same_init(model, gold) -> list:
    """Names of the initial states whose digest differs from the recorded one (empty: bit-identical), or whose set differs."""
    want = {str(k)[len("init_sha256."):]: str(gold[k]) for k in gold.files if str(k).startswith("init_sha256.")}
    got = init_digests(model)
    return sorted(k for k in set(want) | set(got) if want.get(k) != got.get(k))


def trajectory_draws(gold):
    """Every draw of the trajectory in order: batch b's phase is `step<b>_`."""
    return [a for b in range(int(gold["n_steps"])) for a in regenerate(gold, "step%d_" % b)]
