"""Reading LGMRec's golden files (tests/golden/lgmrec_*.npz, written by make_golden_lgmrec.py).

`load`: a setting's file holds only what differs from the file it names in `shared_with` (the default setting); the fields
bit-identical to that file's (the interactions, graphs, the initial weights both settings share, the frozen feature tables)
are read from it.

The random draws: per recorded phase the torch seed, and per draw its kind (Gumbel noise
of `F.gumbel_softmax` or the scaled mask of `F.dropout`), shape, dropout probability and the SHA-256 of its fp32 bytes.  The
draws themselves are regenerated from a CPU `torch.Generator` with that seed: the reference drew them from torch's default
CPU generator seeded the same way and consumed by nothing else within the phase, which make_golden_lgmrec.py asserts by
regenerating every phase and comparing the digests.  (Storing the noise itself would take 4 incompressible bytes per
element: over 2 MB for the H = 64 setting.)"""
import os

import numpy as np
import torch

from golden_io import sha256_fp32


def pack(prefix, seed, specs, draws) -> dict:
    """The fields of one phase: `specs` = [(kind, shape, p)] in draw order, `draws` the arrays drawn."""
    assert len(specs) == len(draws) and all(len(s[1]) == 2 for s in specs)
    return {prefix + "seed": np.int64(seed), prefix + "n_draws": np.int64(len(specs)),
            prefix + "draw_kind": np.array([s[0] for s in specs]), prefix + "draw_shape": np.array([s[1] for s in specs], dtype=np.int64).reshape(-1, 2),
            prefix + "draw_p": np.array([s[2] for s in specs], dtype=np.float64), prefix + "draw_sha256": np.array([sha256_fp32(a) for a in draws])}


def regenerate(gold, prefix):
    """The draws of one phase as fp32 arrays, in order; each checked against its recorded digest."""
    gen = torch.Generator().manual_seed(int(gold[prefix + "seed"]))
    out = []
    for k in range(int(gold[prefix + "n_draws"])):
        kind, shape, p = str(gold[prefix + "draw_kind"][k]), tuple(int(x) for x in gold[prefix + "draw_shape"][k]), float(gold[prefix + "draw_p"][k])
        if kind == "gumbel":                                          # F.gumbel_softmax: -empty_like(logits).exponential_().log()
            x = -torch.empty(shape).exponential_(generator=gen).log()
        else:                                                         # F.dropout (CPU): empty_like(x).bernoulli_(1 - p).div_(1 - p)
            x = torch.empty(shape).bernoulli_(1 - p, generator=gen)
            x.div_(1 - p)
        a = x.numpy()
        assert sha256_fp32(a) == str(gold[prefix + "draw_sha256"][k]), f"{prefix}draw {k}: torch's CPU generator no longer gives the recorded draw"
        out.append(a)
    return out


class Golden:
    """The fields of one setting, `shared_with` resolved; `.files` and `[key]` as an `np.load` result."""

    def __init__(self, path):
        z = np.load(path, allow_pickle=True)
        self._d = {k: z[k] for k in z.files}
        if "shared_with" in self._d:
            base = np.load(os.path.join(os.path.dirname(path), str(self._d["shared_with"])), allow_pickle=True)
            for k in self._d["shared_keys"]:
                self._d[str(k)] = base[str(k)]
        self.files = list(self._d)

    def __getitem__(self, k):
        return self._d[k]


def load(path):
    return Golden(path)


def split_shared(g, base, base_name):
    """`g` without the (non-object) fields bit-identical to those of `base`, plus `shared_with` / `shared_keys`."""
    shared = [k for k, v in g.items() if k in base and v.dtype != object and base[k].dtype != object and v.shape == base[k].shape
              and v.dtype == base[k].dtype and np.array_equal(v, base[k])]
    out = {k: v for k, v in g.items() if k not in shared}
    out["shared_with"], out["shared_keys"] = np.array(base_name), np.array(shared)
    return out
