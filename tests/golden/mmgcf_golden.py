"""Shared by MMGCF's golden generator (make_golden_mmgcf.py), its tests and tools/bench_mmgcf.py: the recorded cases, and
the reference's element-wise fusion as a torch expression, the yardstick of `ops.late_fuse`."""
import torch
import torch.nn.functional as F

from make_golden_mmgcf import CASES, PRUNE_SEED, TRAJ, overrides  # noqa: F401  (re-exported)


def torch_late_fuse(item_e, v, t, fusion, weighting, alpha=None, idx=None):
    """`fuse_item_embeddings` (src/models/mmgcf.py:177-254) for fusion mean | sum, restated on the rows `item_e[idx]`
    with the modality rows v / t (either may be None) and `alpha` = sigmoid(mm_alpha)."""
    e = item_e if idx is None else item_e[idx]
    feats = [f for f in (v, t) if f is not None]

    def apply(ts):
        return torch.stack(ts).mean(dim=0) if fusion == "mean" else torch.stack(ts).sum(dim=0)
    if weighting == "alpha":
        a = alpha.reshape(())
        return apply([e * a] + [f * (1.0 - a) for f in feats])
    if weighting == "normalized":
        return apply([F.normalize(e) * len(feats)] + [F.normalize(f) for f in feats])
    mm = apply(feats) if len(feats) > 1 else feats[0]
    return apply([e, mm])


def grad_errors(gold, grads: dict) -> dict:
    """Per parameter: ||got - ref|| / max(||ref||, 1e-3 * the largest recorded gradient norm), from whole tensors or their
    sketches (a sketch's norm is about sqrt(SKETCH_COLS) times the tensor's).  The projection biases' BPR gradients cancel
    to ~1e-10 (the pos and neg rows carry opposite terms), pure reorder noise: they are measured against the scale of the
    other gradients, not their own."""
    import numpy as np
    import golden_io as G
    pairs = {}
    for k, a in grads.items():
        a = np.asarray(a, dtype=np.float64)
        key = "grad." + k
        if key in gold:
            pairs[k] = (np.asarray(gold[key], dtype=np.float64), a, 1.0)
        else:
            pairs[k] = (np.asarray(gold[key + ".sketch"], dtype=np.float64), G.sketch(a).astype(np.float64), G.SKETCH_COLS ** 0.5)
    scale = max(np.linalg.norm(r) / s for r, _, s in pairs.values())
    return {k: float(np.linalg.norm(g - r) / max(np.linalg.norm(r), 1e-3 * scale * s)) for k, (r, g, s) in pairs.items()}
