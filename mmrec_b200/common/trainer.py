"""Training / evaluation driver with the reference's control flow (`src/common/trainer.py`):
same optimiser construction (`:111-128`), epoch loop with NaN abort and early stopping (`:223-289`) and
evaluation protocol (`:292-311`).  Differences, all on the hot path:

* `evaluate` calls `model.full_sort_topk(batch, k)` -- the fused scoring + mask + top-k kernel path -- when the
  model offers it (`use_fused_topk`, default True); otherwise it takes the reference's dense route
  `full_sort_predict` -> in-place mask -> top-k, through `ops.mask_topk` on CUDA tensors.
* no matplotlib import (the reference's `plot_train_loss`, `:313-332`, is dropped).
"""
import itertools
from logging import getLogger
from time import time

import torch
import torch.optim as optim
from torch.nn.utils.clip_grad import clip_grad_norm_

from ..utils.topk_evaluator import TopKEvaluator
from ..utils.utils import dict2str, early_stopping


class Trainer(object):
    def __init__(self, config, model, mg=False):
        self.config, self.model = config, model
        self.logger = getLogger()
        self.learner = config["learner"]
        self.learning_rate = config["learning_rate"]
        self.epochs = config["epochs"]
        self.eval_step = min(config["eval_step"], self.epochs)
        self.stopping_step = config["stopping_step"]
        self.clip_grad_norm = config["clip_grad_norm"]
        self.valid_metric = config["valid_metric"].lower()
        self.valid_metric_bigger = config["valid_metric_bigger"]
        self.test_batch_size = config["eval_batch_size"]
        self.device = config["device"]
        wd = config["weight_decay"]
        self.weight_decay = 0.0 if wd is None else (eval(wd) if isinstance(wd, str) else wd)
        self.req_training = config["req_training"]
        self.start_epoch, self.cur_step = 0, 0
        zero = {f"{m.lower()}@{k}": 0.0 for m, k in itertools.product(config["metrics"], config["topk"])}
        self.best_valid_score, self.best_valid_result, self.best_test_upon_valid = -1, zero, zero
        self.train_loss_dict = dict()
        self.optimizer = self._build_optimizer()
        sched = config["learning_rate_scheduler"]
        self.lr_scheduler = optim.lr_scheduler.LambdaLR(self.optimizer, lr_lambda=lambda epoch: sched[0] ** (epoch / sched[1]))
        self.evaluator = TopKEvaluator(config)
        self.mg = mg
        self.alpha1, self.alpha2, self.beta = config["alpha1"], config["alpha2"], config["beta"]
        self.use_fused_topk = config["use_fused_topk"] is not False

    def _build_optimizer(self):
        params, lr, wd = list(self.model.parameters()), self.learning_rate, self.weight_decay
        name = self.learner.lower()
        fused = name == "adam" and self.config["fused_adam"] is not False and len(params) > 0 and params[0].is_cuda
        if not fused:
            for p in params:                   # a FusedAdam that owned these parameters before no longer gets factored gradients
                p._mmrec_defer = None
                p._mmrec_pending = None
        if name == "adam":
            # f1: the same optimiser on the kernels of csrc/train.cu (Adam step fused with the projection backward of the
            # trainable modality tables); `config["fused_adam"] = False` keeps torch's.
            if fused:
                from ..optim import FusedAdam
                return FusedAdam(params, lr=lr, weight_decay=wd)
            return optim.Adam(params, lr=lr, weight_decay=wd)
        if name == "sgd":
            return optim.SGD(params, lr=lr, weight_decay=wd)
        if name == "adagrad":
            return optim.Adagrad(params, lr=lr, weight_decay=wd)
        if name == "rmsprop":
            return optim.RMSprop(params, lr=lr, weight_decay=wd)
        self.logger.warning("Received unrecognized optimizer, set default Adam optimizer")
        return optim.Adam(params, lr=lr)

    def _train_epoch(self, train_data, epoch_idx, loss_func=None):
        if not self.req_training:
            return 0.0, []
        self.model.train()
        loss_func = loss_func or self.model.calculate_loss
        total_loss, loss_batches = None, []
        for batch_idx, interaction in enumerate(train_data):
            self.optimizer.zero_grad()
            second_inter = interaction.clone()
            losses = loss_func(interaction)
            if isinstance(losses, tuple):
                loss = sum(losses)
                parts = tuple(l.item() for l in losses)
                total_loss = parts if total_loss is None else tuple(map(sum, zip(total_loss, parts)))
            else:
                loss = losses
                total_loss = losses.item() if total_loss is None else total_loss + losses.item()
            if torch.isnan(loss):
                self.logger.info("Loss is nan at epoch: {}, batch index: {}. Exiting.".format(epoch_idx, batch_idx))
                return loss, torch.tensor(0.0)
            if self.mg and batch_idx % self.beta == 0:          # Mirror Gradient branch (trainer.py:166-183)
                (self.alpha1 * loss).backward()
                self.optimizer.step()
                self.optimizer.zero_grad()
                losses = loss_func(second_inter)
                loss = sum(losses) if isinstance(losses, tuple) else losses
                if torch.isnan(loss):
                    self.logger.info("Loss is nan at epoch: {}, batch index: {}. Exiting.".format(epoch_idx, batch_idx))
                    return loss, torch.tensor(0.0)
                (-1 * self.alpha2 * loss).backward()
            else:
                loss.backward()
            if self.clip_grad_norm:
                if hasattr(self.optimizer, "materialize_pending"):
                    self.optimizer.materialize_pending()        # the norm needs every gradient as a tensor
                clip_grad_norm_(self.model.parameters(), **self.clip_grad_norm)
            self.optimizer.step()
            loss_batches.append(loss.detach())
        return total_loss, loss_batches

    def _valid_epoch(self, valid_data):
        result = self.evaluate(valid_data)
        return (result[self.valid_metric] if self.valid_metric else result["NDCG@20"]), result

    def fit(self, train_data, valid_data=None, test_data=None, saved=False, verbose=True):
        for epoch_idx in range(self.start_epoch, self.epochs):
            t0 = time()
            self.model.pre_epoch_processing()
            train_loss, _ = self._train_epoch(train_data, epoch_idx)
            if torch.is_tensor(train_loss):
                break                                            # NaN loss
            self.lr_scheduler.step()
            self.train_loss_dict[epoch_idx] = sum(train_loss) if isinstance(train_loss, tuple) else train_loss
            t1 = time()
            post_info = self.model.post_epoch_processing()
            if verbose:
                msg = "epoch %d training [time: %.2fs, " % (epoch_idx, t1 - t0)
                if isinstance(train_loss, tuple):
                    msg = ", ".join("train_loss%d: %.4f" % (i + 1, l) for i, l in enumerate(train_loss))
                else:
                    msg += "train loss: %.4f" % train_loss
                self.logger.info(msg + "]")
                if post_info is not None:
                    self.logger.info(post_info)
            if (epoch_idx + 1) % self.eval_step == 0:
                v0 = time()
                valid_score, valid_result = self._valid_epoch(valid_data)
                self.best_valid_score, self.cur_step, stop_flag, update_flag = early_stopping(
                    valid_score, self.best_valid_score, self.cur_step, max_step=self.stopping_step, bigger=self.valid_metric_bigger)
                _, test_result = self._valid_epoch(test_data)
                if verbose:
                    self.logger.info("epoch %d evaluating [time: %.2fs, valid_score: %f]" % (epoch_idx, time() - v0, valid_score))
                    self.logger.info("valid result: \n" + dict2str(valid_result))
                    self.logger.info("test result: \n" + dict2str(test_result))
                if update_flag:
                    if verbose:
                        self.logger.info("██ " + str(self.config["model"]) + "--Best validation results updated!!!")
                    self.best_valid_result, self.best_test_upon_valid = valid_result, test_result
                if stop_flag:
                    if verbose:
                        self.logger.info("+++++Finished training, best eval result in epoch %d" % (epoch_idx - self.cur_step * self.eval_step))
                    break
        return self.best_valid_score, self.best_valid_result, self.best_test_upon_valid

    @torch.no_grad()
    def evaluate(self, eval_data, is_test=False, idx=0):
        from .. import ops
        self.model.eval()
        k = max(self.config["topk"])
        fused = self.use_fused_topk and hasattr(self.model, "full_sort_topk")
        batch_matrix_list = []
        for batched_data in eval_data:
            if fused:
                topk_index = self.model.full_sort_topk(batched_data, k)
            else:
                scores = self.model.full_sort_predict(batched_data)
                _, topk_index = ops.mask_topk(scores, batched_data[1], k)      # trainer.py:305-309
            batch_matrix_list.append(topk_index)
        return self.evaluator.evaluate(batch_matrix_list, eval_data, is_test=is_test, idx=idx)
