"""DygraphModel adapter for FFM (reference: models/rank/ffm/dygraph_model.py:23-98).  Its feeds,
log-loss, AUC metric and train / infer steps are DeepFM's; only the net differs.

Difference kept on purpose (SURVEY.md Q4): Adam updates the fused table lazily (touched rows only);
the reference's dygraph Adam is non-lazy."""
from __future__ import annotations

from ..deepfm.dygraph_model import DygraphModel as _CriteoBase
from . import net


class DygraphModel(_CriteoBase):
    def create_model(self, config):
        """NF = sparse_inputs_slots - 1 + dense_input_dim fields (reference :25-37)."""
        g = config.get
        dense_feature_dim = g("hyper_parameters.dense_input_dim")
        return net.FFMLayer(g("hyper_parameters.sparse_feature_number"),
                            g("hyper_parameters.sparse_feature_dim"), dense_feature_dim,
                            g("hyper_parameters.sparse_inputs_slots") - 1 + dense_feature_dim,
                            device=self.device)
