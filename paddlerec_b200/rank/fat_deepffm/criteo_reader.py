"""FAT-DeepFFM reads the same Criteo slot files as DeepFM (the reference keeps a byte-identical copy
of the reader, and of the sample data, in models/rank/fat_deepffm/)."""
from ..deepfm.criteo_reader import RecDataset  # noqa: F401
