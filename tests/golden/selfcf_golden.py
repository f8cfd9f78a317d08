"""The random draws of SELFCFED_LGN's golden files (tests/golden/selfcfed_lgn_tiny.npz, traj_selfcfed_lgn_tiny.npz;
make_golden_selfcf.py).

A training forward of SELFCFED_LGN draws, in this order: the dropout rate `np.random.random()` of the encoder's
`sparse_dropout` (`src/common/encoders.py:91-93`), `torch.rand(nnz)` on torch's CPU generator (`:79`), then the two
`F.dropout` masks of the targets, users first (`src/models/selfcfed_lgn.py:42-47`).  The reference ran on the CPU, so all
three come from the seeded CPU generators.  A phase keeps the numpy and torch seed it started from and the SHA-256 of each
draw; `Replay` regenerates them by consuming the same generators in the same order: `np.random.random()` and `torch.rand` are
the encoder's own calls, and `F.dropout` becomes torch's CPU expression (`empty_like(x).bernoulli_(1 - p).div_(1 - p)`) on
the CPU generator, moved to the device.  (A model on the GPU would draw its target masks from the device generator.)"""
import numpy as np
import torch
import torch.nn.functional as F

from golden_io import sha256_fp32


def cpu_dropout_mask(shape, p):
    """`F.dropout`'s scaled keep mask as torch draws it on the CPU (the default generator)."""
    m = torch.empty(shape).bernoulli_(1 - p)
    return m.div_(1 - p)


class Replay:
    """Seeds a phase and makes `F.dropout` draw its masks on the CPU generator as the reference's CPU run did.  `digests`
    collects the SHA-256 of every draw of the phase in order: `torch.rand` (the encoder's dropout draws) and the masks."""

    def __init__(self, seed):
        self.seed, self.digests = int(seed), []
        self._saved = None

    def seed_phase(self):
        np.random.seed(self.seed)
        torch.manual_seed(self.seed)

    def dropout(self, input, p=0.5, training=True, inplace=False):
        assert not inplace
        if not training or p == 0 or input.numel() == 0:
            return input
        m = cpu_dropout_mask(tuple(input.shape), p)
        self.digests.append(sha256_fp32(m.numpy()))
        return input * m.to(input.device)

    def rand(self, *size, **kw):
        x = self._rand(*size, **kw)
        if x.device.type == "cpu" and x.dtype == torch.float32:
            self.digests.append(sha256_fp32(x.numpy()))
        return x

    def __enter__(self):
        self._saved = (F.dropout, torch.rand)
        self._rand = torch.rand
        F.dropout, torch.rand = self.dropout, self.rand
        self.seed_phase()
        return self

    def __exit__(self, *exc):
        F.dropout, torch.rand = self._saved

