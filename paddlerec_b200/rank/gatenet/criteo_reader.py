"""GateNet reads the same Criteo slot files as DeepFM (the reference keeps a byte-identical copy of the
reader, and of the sample data, in models/rank/gatenet/)."""
from ..deepfm.criteo_reader import RecDataset  # noqa: F401
