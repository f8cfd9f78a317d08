"""Shared by VBPR's and BPR's tests and tools/bench_vbpr.py: the reference's loss after the tables as a torch expression,
the yardstick of `ops.bpr_mf_loss`."""
import torch

from make_golden_vbpr import CASES, TRAJ  # noqa: F401  (re-exported)


def torch_bpr_mf_loss(U, A, P, users, pos, neg, reg_weight):
    """`calculate_loss` of src/models/vbpr.py:85-98 / bpr.py:75-87 from the gathered rows: user_e = U[users], the item
    rows [A[pos] | P[:B]] and [A[neg] | P[B:]] (P None: A's rows alone), `BPRLoss` + reg_weight * `EmbLoss`."""
    from mmrec_b200.common.loss import BPRLoss, EmbLoss
    B = users.numel()
    user_e, pos_e, neg_e = U[users, :], A[pos, :], A[neg, :]
    if P is not None:
        pos_e, neg_e = torch.cat((pos_e, P[:B]), -1), torch.cat((neg_e, P[B:]), -1)
    pos_item_score, neg_item_score = torch.mul(user_e, pos_e).sum(dim=1), torch.mul(user_e, neg_e).sum(dim=1)
    mf_loss = BPRLoss()(pos_item_score, neg_item_score)
    reg_loss = EmbLoss()(user_e, pos_e, neg_e)
    return mf_loss + reg_weight * reg_loss
