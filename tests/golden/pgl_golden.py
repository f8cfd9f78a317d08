"""Shared by PGL's tests and tools/bench_pgl.py: the reference's loss after the tables as a torch expression, the yardstick
of `ops.pgl_loss`, and the recorded dropout masks."""
import numpy as np
import torch
import torch.nn.functional as F

from make_golden_pgl import LOSS_SEED, PRUNE_SEED, REG_CASES, TRAJ_OVER, TRAJ_SEED0  # noqa: F401  (re-exported)


def masks_of(gold):
    """The four recorded bool masks [4, B, 2d] of one `calculate_loss` (views a, b, c, d)."""
    shape = tuple(int(x) for x in gold["masks_shape"])
    return torch.from_numpy(np.unpackbits(gold["masks"], axis=-1, count=shape[-1]).astype(bool).reshape(shape))


def cpu_drop(x, m, p):
    """The reference's CPU dropout with the mask m: `x * (noise / (1 - p))`."""
    return x * m.to(x.dtype).div(1 - p)


def info_nce(view1, view2, temperature=0.2, ttl_fn=None):
    """`InfoNCE` of src/models/pgl.py:240-248; `ttl_fn(v1, v2, tau)` replaces the [B, B] exp-sum (e.g. ops.expsum_rows)."""
    view1, view2 = F.normalize(view1, dim=1), F.normalize(view2, dim=1)
    pos_score = (view1 * view2).sum(dim=-1)
    pos_score = torch.exp(pos_score / temperature)
    if ttl_fn is None:
        ttl_score = torch.matmul(view1, view2.transpose(0, 1))
        ttl_score = torch.exp(ttl_score / temperature).sum(dim=1)
    else:
        ttl_score = ttl_fn(view1, view2, temperature)
    cl_loss = -torch.log(pos_score / ttl_score)
    return torch.mean(cl_loss)


def torch_pgl_loss(UA, IA, users, pos, neg, masks, dropout, reg_weight, drop=cpu_drop, ttl_fn=None):
    """`calculate_loss` of src/models/pgl.py:250-259 after `forward`: the gathers, `bpr_loss`, the four dropout views (in the
    order a, b, c, d, each `drop(rows, mask, dropout)`; masks None: the rows themselves) and the two InfoNCE terms."""
    u, p, n = UA[users], IA[pos], IA[neg]
    pos_scores = torch.sum(torch.mul(u, p), dim=1)
    neg_scores = torch.sum(torch.mul(u, n), dim=1)
    mf_loss = -torch.mean(F.logsigmoid(pos_scores - neg_scores))
    if masks is None:
        a, b, c, d = u, u, p, p
    else:
        a, b = drop(u, masks[0], dropout), drop(u, masks[1], dropout)
        c, d = drop(p, masks[2], dropout), drop(p, masks[3], dropout)
    cl_loss = (info_nce(a, b, ttl_fn=ttl_fn) + info_nce(c, d, ttl_fn=ttl_fn)) / 2
    return mf_loss + reg_weight * cl_loss


class DeviceDropout(torch.autograd.Function):
    """torch's dropout on the device with a given mask: forward (x * m) * scale, backward (g * m) * scale_bwd
    (`native_dropout` / `native_dropout_backward`)."""

    @staticmethod
    def forward(ctx, x, m, p):
        from mmrec_b200.ops import dropout_scales
        sf, sb = dropout_scales(p)
        ctx.save_for_backward(m)
        ctx.sb = sb
        return (x * m.to(x.dtype)) * sf

    @staticmethod
    def backward(ctx, g):
        m, = ctx.saved_tensors
        return (g * m.to(g.dtype)) * ctx.sb, None, None


def device_drop(x, m, p):
    return DeviceDropout.apply(x, m, p)


def reference_calculate_loss(model, interaction, adj=None):
    """`calculate_loss` of src/models/pgl.py:250-259 as the reference's own expressions (its `bpr_loss`, its four
    `self.dropoutf` calls, its InfoNCE) on the model's `forward`: the generator advances as the reference's does."""
    users, pos_items, neg_items = interaction[0], interaction[1], interaction[2]
    ua, ia = model.forward(model.sub_graph if adj is None else adj)
    u, p, n = ua[users], ia[pos_items], ia[neg_items]
    pos_scores = torch.sum(torch.mul(u, p), dim=1)
    neg_scores = torch.sum(torch.mul(u, n), dim=1)
    mf_loss = -torch.mean(F.logsigmoid(pos_scores - neg_scores))
    cl_loss = (info_nce(model.dropoutf(u), model.dropoutf(u)) + info_nce(model.dropoutf(p), model.dropoutf(p))) / 2
    return mf_loss + model.reg_weight * cl_loss
