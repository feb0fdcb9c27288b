"""DygraphModel adapter for FAT-DeepFFM (reference: models/rank/fat_deepffm/dygraph_model.py:23-98).
Its feeds, log-loss, AUC metric and train / infer steps are DeepFM's; only the net differs.

Difference kept on purpose (SURVEY.md Q4, Q17): Adam updates the fused table lazily (touched rows
only); the reference's dygraph Adam is non-lazy."""
from __future__ import annotations

from ..deepfm.dygraph_model import DygraphModel as _CriteoBase
from . import net


class DygraphModel(_CriteoBase):
    def create_model(self, config):
        """sparse_num_field = sparse_inputs_slots - 1 (the label is a slot; reference :25-37)."""
        g = config.get
        return net.FAT_DeepFFMLayer(g("hyper_parameters.sparse_feature_number"),
                                    g("hyper_parameters.sparse_feature_dim"),
                                    g("hyper_parameters.dense_input_dim"),
                                    g("hyper_parameters.sparse_inputs_slots") - 1,
                                    g("hyper_parameters.layer_sizes_dnn"), device=self.device)
