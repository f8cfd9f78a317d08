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

from golden_io import sha256_fp32


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
        assert sha256_fp32(a) == str(gold[prefix + "draw_sha256"][k]), f"{prefix}draw {k}: torch's CPU generator no longer gives the recorded draw"
        out.append(a)
    return out


def plain(model) -> dict:
    """The plain tensors the reference keeps beside its parameters, whose initial digests the files keep as
    `init_sha256.plain.<name>` (`golden_io.init_digests`): not the 1.2 MiB of incompressible weights."""
    out = {"collaborative": model.collaborative}
    for m in "vtc":
        out["%s_preference" % m] = getattr(model, m + "_gcn").preference
    out["result_embed0"] = model.result_embed
    return out


def trajectory_draws(gold):
    """Every draw of the trajectory in order: batch b's phase is `step<b>_`."""
    return [a for b in range(int(gold["n_steps"])) for a in regenerate(gold, "step%d_" % b)]
