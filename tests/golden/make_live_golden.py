"""Mints tests/golden/reference_live_<tag>.npz (and copies the reference's bundled sample files next
to them) by EXECUTING THE REFERENCE'S OWN CODE, unmodified, on top of oracle/paddle_shim.py:

  models/rank/{deepfm,dcn_v2,wide_deep,din,dlrm}/net.py   float64 forward of small seeded layers: the
                                                           parameters (rounded to float32 values, so
                                                           they are stored exactly in half the bytes),
                                                           the inputs, the output and the gradient of
                                                           sum(out^2) w.r.t. every parameter
  models/rank/{deepfm,dcn_v2}/*reader.py, din/dinReader.py what the readers yield for their sample files

tests/test_oracle_reference_live.py replays every case against oracle/nets.py, oracle/readers.py and
the native parsers without the reference checkout.  Usage (needs a PaddleRec checkout):

    python tests/golden/make_live_golden.py <path of the PaddleRec checkout>
"""
import gzip
import importlib.util
import os
import shutil
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import paddle_shim  # noqa: E402

OUT = {}   # {file tag: {key: array}}


def _grads(loss, named):
    gs = torch.autograd.grad(loss, list(named.values()), allow_unused=True, retain_graph=True)
    return {k: (torch.zeros_like(p) if g is None else g) for (k, p), g in zip(named.items(), gs)}


def rounded(layer, extra=()):
    with torch.no_grad():
        for p in list(layer.parameters()) + list(extra):
            p.copy_(p.float().double())
    return layer


def record(case, named, out, inputs):
    """Parameters (aliases of one tensor stored once), inputs, output, gradients of sum(out^2)."""
    tag = case.split("_")[0]
    dst = OUT.setdefault(tag, {})
    uniq = []
    for k, p in named.items():
        idx = next((i for i, q in enumerate(uniq) if q is p), None)
        if idx is None:
            uniq.append(p)
            idx = len(uniq) - 1
        dst["%s/param/%s" % (case, k)] = np.asarray(idx)
    for i, p in enumerate(uniq):
        dst["%s/tensor/%d" % (case, i)] = p.detach().float().numpy()
    for k, v in inputs.items():
        dst["%s/input/%s" % (case, k)] = v.numpy()
    dst["%s/out" % case] = out.detach().numpy()
    for k, g in _grads(out.square().sum(), named).items():
        dst["%s/grad/%s" % (case, k)] = g.numpy()


def slots(ids):
    return {"ids": torch.cat(ids, 1)}


def nets(ref_root):
    torch.set_default_dtype(torch.float64)
    for seed, D, B in [(1, 5, 3), (2, 12, 9)]:
        ref = paddle_shim.import_reference_net("deepfm", ref_root)
        torch.manual_seed(seed)
        V, fc = 61, [7, 5, 3]
        layer = rounded(ref.DeepFMLayer(V, D, 13, 26, fc))
        ids = [torch.randint(0, V, (B, 1)) for _ in range(26)]
        dense = torch.rand(B, 13)
        record("deepfm_%d_%d_%d" % (seed, D, B), dict(layer.named_parameters()), layer(ids, dense),
               dict(slots(ids), dense=dense))
    for mix, stacked in [(False, False), (True, True)]:
        ref = paddle_shim.import_reference_net("dcn_v2", ref_root)
        torch.manual_seed(11)
        V, D, B, fc = 43, 3, 5, [9, 6]
        layer = rounded(ref.DCN_V2Layer(V, D, 13, 26, fc, 3, stacked, mix, 4, 2))
        layer.eval()
        ids = [torch.randint(0, V, (B, 1)) for _ in range(26)]
        dense = torch.rand(B, 13)
        record("dcn_v2_%d_%d" % (mix, stacked), dict(layer.named_parameters()), layer(ids, dense),
               dict(slots(ids), dense=dense))
    torch.manual_seed(5)
    ref = paddle_shim.import_reference_net("wide_deep", ref_root)
    V, D, B, fc = 37, 6, 4, [8, 4]
    layer = rounded(ref.WideDeepLayer(V, D, 13, 26, fc))
    ids = [torch.randint(0, V, (B, 1)) for _ in range(26)]
    dense = torch.rand(B, 13)
    record("wide_deep", dict(layer.named_parameters()), layer(ids, dense), dict(slots(ids), dense=dense))
    refd = paddle_shim.import_reference_net("din", ref_root)
    layer = rounded(refd.DINLayer(4, 4, "sigmoid", False, False, 29, 7))
    B, L = 3, 5
    hi, hc = torch.randint(0, 29, (B, L)), torch.randint(0, 7, (B, L))
    ti, tc = torch.randint(0, 29, (B,)), torch.randint(0, 7, (B,))
    mask = torch.zeros(B, L, 1, dtype=torch.int64)
    mask[1, 3:] = int(-1e9)
    named = dict(layer.named_parameters())
    for i, m in enumerate([m for m in layer.attention_layer if hasattr(m, "weight")]):
        named["att.linear_%d.weight" % i], named["att.linear_%d.bias" % i] = m.weight, m.bias
    rounded(layer, named.values())   # the attention linears are not among layer.parameters()
    args = (hi, hc, ti, tc, None, mask, ti.unsqueeze(1).repeat(1, L), tc.unsqueeze(1).repeat(1, L))
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp())                 # the reference may write ./tmp.txt
    try:
        out = layer(*args)
    finally:
        os.chdir(cwd)
    record("din", named, out, dict(hi=hi, hc=hc, ti=ti, tc=tc, mask=mask))
    for self_interaction, B, d in [(False, 6, 4), (True, 9, 8)]:
        ref = paddle_shim.import_reference_net("dlrm", ref_root)
        torch.manual_seed(21 + B)
        V, bot, top = 53, [10, d], [12, 2]
        layer = rounded(ref.DLRMLayer(13, bot, V, d, top, 26, self_interaction=self_interaction))
        layer.train()
        ids = [torch.randint(0, V, (B, 1)) for _ in range(26)]
        dense = torch.rand(B, 13)
        record("dlrm_%d_%d_%d" % (self_interaction, B, d), dict(layer.named_parameters()),
               layer(ids, dense), dict(slots(ids), dense=dense))
    torch.set_default_dtype(torch.float32)


def readers(ref_root):
    paddle_shim.install()
    R = OUT.setdefault("readers", {})
    rank = os.path.join(ref_root, "models", "rank")

    def load(path, name):
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod

    sample = os.path.join(rank, "deepfm/data/sample_data/train/sample_train.txt")
    with open(sample, "rb") as src, gzip.GzipFile(os.path.join(HERE, "ref_deepfm_sample_train.txt.gz"),
                                                  "wb", mtime=0) as dst:
        dst.write(src.read())
    ds = load(os.path.join(rank, "deepfm/criteo_reader.py"), "ref_criteo_reader").RecDataset([sample], None)
    ds.inference = False
    rows = list(ds)
    R["reader/deepfm/ids"] = np.stack([np.concatenate(r[:27]) for r in rows])
    R["reader/deepfm/dense"] = np.stack([r[27] for r in rows])

    dcn_sample = os.path.join(rank, "dcn_v2/data/sample_data/sample_train.txt")
    assert open(dcn_sample, "rb").read() == open(sample, "rb").read()   # one file serves both
    rows = list(load(os.path.join(rank, "dcn_v2/reader.py"), "ref_dcn_reader").RecDataset([dcn_sample], None))
    R["reader/dcn_v2/ids"] = np.stack([np.concatenate(r[1:27]) for r in rows])
    R["reader/dcn_v2/dense"] = np.stack([r[27] for r in rows])

    din_sample = os.path.join(rank, "din/data/train_data/sample_data.txt")
    shutil.copyfile(din_sample, os.path.join(HERE, "ref_din_sample_data.txt"))
    cwd = os.getcwd()
    os.chdir(tempfile.mkdtemp())                 # dinReader.py writes ./tmp.txt
    try:
        rd = load(os.path.join(rank, "din/dinReader.py"), "ref_din_reader")
        samples = list(rd.RecDataset([din_sample], {"runner.train_batch_size": 8}))
    finally:
        os.chdir(cwd)
    R["reader/din/n_samples"] = np.asarray(len(samples))
    for b in range(len(samples) // 8):
        for j in range(len(samples[0])):
            R["reader/din/%d/%d" % (b, j)] = np.stack([np.asarray(s[j]) for s in samples[8 * b:8 * b + 8]])


if __name__ == "__main__":
    ref_root = os.path.abspath(sys.argv[1])
    nets(ref_root)
    readers(ref_root)
    for tag, arrays in OUT.items():
        np.savez_compressed(os.path.join(HERE, "reference_live_%s.npz" % tag), **arrays)
    print("wrote", sorted(OUT))
