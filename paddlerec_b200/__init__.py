"""paddlerec_b200 — H100-native sparse-embedding + feature-interaction engine behind PaddleRec's
rank-model surface (models/rank/*/net.py, DygraphModel).  See DESIGN.md.

  csrc/            hand-written sm_90a CUDA kernels + the C ABI (include/b200rec.h)
  _lib.py          ctypes binding / in-tree nvcc build of lib/libb200rec.so
  ops.py           torch wrappers of the C ABI + autograd glue (SelectedRows gradients)
  nn.py            Embedding / Linear with Paddle's semantics
  optim.py         Adam(lazy) / SGD / row-wise AdaGrad over SelectedRows
  sharded.py       row-cyclic table sharding over NCCL all-to-all
  rank/<model>/    net.py + dygraph_model.py mirrors of the reference's plugin directories
  dataio.py        native text parsers (include/b200rec_io.h) + PackedBatchReader
  checkpoint.py    rec.pdparams in paddle.save's pickle layout, rec.pdopt for resume
  runner.py        tools/trainer.py-shaped loop and yaml loader
"""
__version__ = "0.1.0"
