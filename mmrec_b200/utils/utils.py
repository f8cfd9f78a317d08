"""Small helpers with the reference's behaviour (`src/utils/utils.py:17-116`)."""
import datetime
import importlib
import random

import numpy as np
import torch


def get_local_time():
    return datetime.datetime.now().strftime("%b-%d-%Y-%H-%M-%S")


def get_model(model_name):
    """`models/<lowercase name>.py`, class `<name>` -- the reference's plugin loader (`utils.py:28-41`)."""
    module = importlib.import_module("mmrec_b200.models." + model_name.lower())
    return getattr(module, model_name)


def get_trainer():
    return getattr(importlib.import_module("mmrec_b200.common.trainer"), "Trainer")


def init_seed(seed):
    random.seed(seed)
    np.random.seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(seed)
        torch.cuda.manual_seed_all(seed)
    torch.manual_seed(seed)


def early_stopping(value, best, cur_step, max_step, bigger=True):
    stop_flag, update_flag = False, False
    better = value > best if bigger else value < best
    if better:
        cur_step, best, update_flag = 0, value, True
    else:
        cur_step += 1
        stop_flag = cur_step > max_step
    return best, cur_step, stop_flag, update_flag


def dict2str(result_dict):
    return "".join(str(m) + ": " + "%.04f" % v + "    " for m, v in result_dict.items())
