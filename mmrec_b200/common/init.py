"""Parameter initialisation with the reference's semantics (`src/common/init.py:8-24`): the models that call
`self.apply(xavier_normal_initialization)` draw the same numbers in the same order, so `init_seed` gives the reference's
initial weights bit for bit."""
import torch.nn as nn
from torch.nn.init import constant_, xavier_normal_


def xavier_normal_initialization(module):
    """`xavier_normal_` of the weight of every `nn.Embedding` and `nn.Linear`, and a zero bias for `nn.Linear`."""
    if isinstance(module, nn.Embedding):
        xavier_normal_(module.weight.data)
    elif isinstance(module, nn.Linear):
        xavier_normal_(module.weight.data)
        if module.bias is not None:
            constant_(module.bias.data, 0)
