"""DygraphModel adapter for GateNet (reference: models/rank/gatenet/dygraph_model.py:23-100).  Its
feeds, log-loss, AUC metric and train / infer steps are DeepFM's; only the net differs.

Difference kept on purpose (SURVEY.md Q4, Q18): Adam updates the table lazily (touched rows only);
the reference's dygraph Adam is non-lazy.  `sparse_fea_num` is read by the reference and never
used; it is not read here."""
from __future__ import annotations

from ..deepfm.dygraph_model import DygraphModel as _CriteoBase
from . import net


class DygraphModel(_CriteoBase):
    def create_model(self, config):
        """num_field = sparse_inputs_slots - 1 (the label takes one slot; reference :25-41)."""
        g = config.get
        return net.GateDNNLayer(g("hyper_parameters.sparse_feature_number"),
                                g("hyper_parameters.sparse_feature_dim"),
                                g("hyper_parameters.dense_input_dim"),
                                g("hyper_parameters.sparse_inputs_slots") - 1,
                                g("hyper_parameters.fc_sizes"),
                                g("hyper_parameters.use_embedding_gate"),
                                g("hyper_parameters.use_hidden_gate"), device=self.device)
