"""DygraphModel adapter for ESMM — the reference's plugin surface
(models/multitask/esmm/dygraph_model.py:23-114): the same seven methods with the same argument
meaning, over CUDA tensors and the b200rec kernels.

Differences that are deliberate (SURVEY.md Q4, Q19):
  * create_feeds makes ONE [B,23,max_len] int64 copy and the two label copies instead of 25 copies;
  * the two AUC metrics keep their histograms on the device (no `.numpy()` sync per step);
  * Adam updates the table lazily (touched rows only); the reference's dygraph Adam is non-lazy.
"""
from __future__ import annotations

import numpy as np
import torch

from ... import functional as BF
from ... import optim
from . import net


def _to_host_tensor(b):
    if isinstance(b, torch.Tensor):
        return b
    return torch.from_numpy(np.asarray(b))


class DygraphModel:
    device = "cuda"

    def create_model(self, config):
        """The yaml's hyper_parameters -> ESMMLayer on `self.device` (reference :25-40)."""
        g = config.get
        return net.ESMMLayer(g("hyper_parameters.sparse_feature_number"),
                             g("hyper_parameters.sparse_feature_dim"),
                             g("hyper_parameters.num_field"),
                             g("hyper_parameters.ctr_fc_sizes"),
                             g("hyper_parameters.cvr_fc_sizes"), device=self.device)

    def create_feeds(self, batch_data, config):
        """batch_data: the reader's 23 [B, max_len] id arrays then [B,1] click and [B,1] buy (host
        arrays or tensors), or the packed form (ids [B,23,max_len], click [B,1], buy [B,1]).
        Returns (ids [B,23,max_len] int64, ctr_label [B,1] int64, ctcvr_label [B,1] int64)."""
        max_len = int(config.get("hyper_parameters.max_len", 3))
        if len(batch_data) == 3:
            ids, clk, buy = (_to_host_tensor(b) for b in batch_data)
        else:
            ids = torch.stack([_to_host_tensor(b).reshape(-1, max_len) for b in batch_data[:-2]], 1)
            clk, buy = _to_host_tensor(batch_data[-2]), _to_host_tensor(batch_data[-1])
        dev = self.device
        ids = ids.to(torch.int64).to(dev, non_blocking=True)
        clk = clk.reshape(-1, 1).to(torch.int64).to(dev, non_blocking=True)
        buy = buy.reshape(-1, 1).to(torch.int64).to(dev, non_blocking=True)
        return ids, clk, buy

    def create_loss(self, ctr_out_one, ctr_clk, ctcvr_prop_one, ctcvr_buy):
        """mean(log_loss(ctr_one, clk) + log_loss(ctcvr_one, buy)), Paddle's epsilon 1e-4
        (reference :56-67): the mean of a sum is the sum of the two means."""
        return BF.log_loss_mean(ctr_out_one, ctr_clk) + BF.log_loss_mean(ctcvr_prop_one, ctcvr_buy)

    def create_optimizer(self, dy_model, config):
        """Adam over every parameter; the table is updated row-wise from its SelectedRows gradient
        (lazy_mode — the reference's dygraph Adam :70-74 is non-lazy)."""
        lr = config.get("hyper_parameters.optimizer.learning_rate", 0.001)
        return optim.Adam(learning_rate=lr, parameters=dy_model.parameters(), lazy_mode=True)

    def create_metrics(self):
        """Two ROC-AUC metrics, auc_ctr and auc_ctcvr (reference :78-83), on the device."""
        return [BF.Auc("ROC"), BF.Auc("ROC")], ["auc_ctr", "auc_ctcvr"]

    def train_forward(self, dy_model, metrics_list, batch_data, config):
        """-> (loss, metrics_list, print_dict) (reference :86-101): auc_ctr on ctr_out, auc_ctcvr on
        ctcvr_prop, both read without leaving the device."""
        ids, label_ctr, label_ctcvr = self.create_feeds(batch_data, config)
        ctr_out, ctr_one, _, _, ctcvr_prop, ctcvr_one = dy_model.forward(ids)
        loss = self.create_loss(ctr_one, label_ctr, ctcvr_one, label_ctcvr)
        if metrics_list:
            metrics_list[0].update(preds=ctr_out.detach(), labels=label_ctr)
            metrics_list[1].update(preds=ctcvr_prop.detach(), labels=label_ctcvr)
        return loss, metrics_list, {"loss": loss}

    def infer_forward(self, dy_model, metrics_list, batch_data, config):
        """-> (metrics_list, None): forward under no_grad + the two metric updates (:103-114)."""
        ids, label_ctr, label_ctcvr = self.create_feeds(batch_data, config)
        with torch.no_grad():
            ctr_out, _, _, _, ctcvr_prop, _ = dy_model.forward(ids)
        if metrics_list:
            metrics_list[0].update(preds=ctr_out, labels=label_ctr)
            metrics_list[1].update(preds=ctcvr_prop, labels=label_ctcvr)
        return metrics_list, None
