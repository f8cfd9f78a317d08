"""Loss modules with the reference's semantics (`src/common/loss.py:9-62`); plain torch, not on
the kernel path (SURVEY.md 2.1 #9)."""
import torch
import torch.nn as nn


class BPRLoss(nn.Module):
    def __init__(self, gamma=1e-10):
        super().__init__()
        self.gamma = gamma

    def forward(self, pos_score, neg_score):
        return -torch.log(self.gamma + torch.sigmoid(pos_score - neg_score)).mean()


class EmbLoss(nn.Module):
    def __init__(self, norm=2):
        super().__init__()
        self.norm = norm

    def forward(self, *embeddings):
        out = torch.zeros(1, device=embeddings[-1].device)
        for e in embeddings:
            out = out + torch.norm(e, p=self.norm)
        return out / embeddings[-1].shape[0]


class L2Loss(nn.Module):
    def forward(self, *embeddings):
        out = torch.zeros(1, device=embeddings[-1].device)
        for e in embeddings:
            out = out + torch.sum(e ** 2) * 0.5
        return out
