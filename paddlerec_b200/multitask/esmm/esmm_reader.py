"""Ali-CCP sample reader for ESMM, restating the reference's models/multitask/esmm/esmm_reader.py
(RecDataset :21-76).  A line is `sample_id,click,buy,<skipped>,field:feat,...`:

  * the fourth column is never read (the reference parses features from column 4 on);
  * a feature whose field is not one of the 23 below is dropped;
  * each field keeps its first `max_len` ids in line order and is padded with id 0;
  * a sample is 23 int64 arrays of length max_len, then [click] and [buy], in file and line order.

`hyper_parameters.max_len` defaults to 3; the reference's config.yaml does not set it.
"""
from __future__ import annotations

import numpy as np
import torch

FIELDS = ("101", "109_14", "110_14", "127_14", "150_14", "121", "122", "124", "125", "126", "127",
          "128", "129", "205", "206", "207", "210", "216", "508", "509", "702", "853", "301")
PADDING = 0


def parse_line(line: str, max_len: int):
    """One CSV line -> 23 int64 [max_len] id arrays, then [click], [buy]."""
    cols = line.strip().split(",")
    bags = {f: [] for f in FIELDS}
    for elem in cols[4:]:
        field, feat = elem.strip().split(":")
        if field in bags:
            bags[field].append(int(feat))
    out = []
    for f in FIELDS:
        ids = bags[f][:max_len]
        out.append(np.array(ids + [PADDING] * (max_len - len(ids)), dtype=np.int64))
    out.append(np.array([int(cols[1])], dtype=np.int64))
    out.append(np.array([int(cols[2])], dtype=np.int64))
    return out


class RecDataset(torch.utils.data.IterableDataset):
    def __init__(self, file_list, config):
        super().__init__()
        self.file_list = file_list
        self.max_len = int(config.get("hyper_parameters.max_len", 3))

    def __iter__(self):
        for path in self.file_list:
            with open(path, "r") as fh:
                for line in fh:
                    yield parse_line(line, self.max_len)
