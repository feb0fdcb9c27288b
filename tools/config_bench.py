#!/usr/bin/env python
"""BASELINE.json configs 3, 4 and 5 on N GPUs of one box (one process per GPU; N=1 runs plain):

    python tools/config_bench.py --what dcn|din|gather [...]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \\
        --master-port 29511 tools/config_bench.py --what dcn

  dcn     config 3: DCN-V2 Criteo-shape (D=40, CrossNetV2 x2 on the wgmma kernels, fc [768,768],
          Adam + global-norm clip), embedding table row-sharded (id mod N) with the NCCL all-to-all
          exchange, dense parameters data-parallel; weak scaling, B per GPU fixed.
  din     config 4: DIN AmazonElec-shape (63001 items / 801 cats, E=64+64, history 100): tables are
          tiny -> replicas only: N independent replicas, no collective (DESIGN.md section 5).
  gather  config 5: Wide&Deep lookup sweep, V in {1e6..1e9} x D in {16,64,128}: the sharded lookup
          (bucketize -> ids all-to-all -> owner b200rec_gather -> rows all-to-all -> unpermute),
          reported as useful gather GB/s over ALL GPUs: B*26*(8 + 2*4*D) algorithmic bytes per GPU
          per step (SURVEY.md 8(d)); tables that exceed one GPU's HBM only run where they fit.

Every line is one JSON object; times are CUDA events, max over ranks.  Synthetic data, seed 12345.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch.distributed as dist  # noqa: E402


def setup():
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    return rank, world, torch.device("cuda", local)


def timed(fn, iters, warm, world, dev):
    for i in range(warm):
        fn(i)
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fn(warm + i)
    e1.record()
    if world > 1:
        dist.barrier()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    return ms


def emit(rank, obj):
    if rank == 0:
        print(json.dumps(obj), flush=True)


def criteo_batches(n, B, V, seed, dev, log_dense=False):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        ids = torch.randint(1, V, (B, 26), generator=g)
        ids[torch.rand(B, 26, generator=g) < 0.02] = 0
        dense = torch.rand(B, 13, generator=g)
        if log_dense:
            dense = torch.log1p(dense * 10)
        label = (torch.rand(B, 1, generator=g) < 0.29).long()
        out.append(tuple(t.to(dev) for t in (label, ids, dense)))
    return out


def run_dcn(a, rank, world, dev):
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200 import sharded
    from paddlerec_b200.rank.dcn_v2.dygraph_model import DygraphModel
    bnn.set_matmul_precision("bf16x3")
    cfg = {"hyper_parameters.sparse_feature_number": a.V, "hyper_parameters.sparse_feature_dim": a.D,
           "hyper_parameters.fc_sizes": [768, 768], "hyper_parameters.dense_input_dim": 13,
           "hyper_parameters.sparse_inputs_slots": 27, "hyper_parameters.cross_num": 2,
           "hyper_parameters.is_Stacked": True, "hyper_parameters.use_low_rank_mixture": False,
           "hyper_parameters.low_rank": 256, "hyper_parameters.num_experts": 4,
           "hyper_parameters.optimizer.learning_rate": 1e-4}
    torch.manual_seed(12345)
    dm = DygraphModel()
    dm.device = dev
    if world > 1:
        # build the table shard directly (a replicated 1e8 x 40 table would be 16 GB per rank)
        from paddlerec_b200.rank.dcn_v2 import net
        small = dict(cfg)
        small["hyper_parameters.sparse_feature_number"] = 8
        model = dm.create_model(small)
        std = 0.1 / a.D ** 0.5
        model.embedding = sharded.ShardedEmbedding(a.V, a.D, 0, rank, world, init_std=std, device=dev)
        sharded.sync_dense_parameters(model)
        opt = sharded.DistributedOptimizer(dm.create_optimizer(model, cfg), model, world)
    else:
        model = dm.create_model(cfg)
        opt = dm.create_optimizer(model, cfg)
    model.eval()        # Dropout(0.5) off: the deterministic path, same kernels
    batches = criteo_batches(4, a.B, a.V, 12345 + rank, dev, log_dense=True)
    scale = opt.scale_loss if hasattr(opt, "scale_loss") else (lambda x: x)

    def step(i):
        opt.clear_grad()
        loss, _, _ = dm.train_forward(model, None, batches[i % 4], cfg)
        scale(loss).backward()
        opt.step()
    ms = timed(step, a.iters, 3, world, dev)
    C = 39 * a.D
    flops = 3 * 3 * 2.0 * a.B * (2 * C * C + C * 768 + 768 * 768)      # bf16x3, fwd + dX + dW
    emit(rank, {"config": 3, "what": "DCN-V2 Criteo-shape train step (stacked, CrossNetV2 x2 on the "
                "tcgen05 GEMMs, fc [768,768], Adam + global-norm clip)", "n_gpus": world,
                "B_per_gpu": a.B, "V": a.V, "D": a.D, "ms_per_step": ms,
                "samples_per_s": a.B * world / ms * 1e3, "scaling": "weak",
                "parallelism": "single GPU" if world == 1 else
                "table row-sharded (id mod %d) + NCCL all-to-all; dense data-parallel" % world,
                "tower_gemm_tflops_lower_bound": round(flops / (ms / 1e3) / 1e12, 1)})


def run_din(a, rank, world, dev):
    from paddlerec_b200 import nn as bnn
    from paddlerec_b200.rank.din.dygraph_model import DygraphModel
    bnn.set_matmul_precision("bf16x3")
    B, L = a.B, a.L
    g = torch.Generator().manual_seed(12345 + rank)
    dm = DygraphModel()
    dm.device = dev
    cfg = {"hyper_parameters.item_count": 63001, "hyper_parameters.cat_count": 801,
           "hyper_parameters.optimizer.learning_rate_base_lr": 0.85}
    torch.manual_seed(12345)
    model = dm.create_model(cfg)
    opt = dm.create_optimizer(model, cfg)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    hi = torch.randint(1, 63001, (B, L), generator=g)
    hc = torch.randint(1, 801, (B, L), generator=g)
    mask = torch.zeros(B, L, 1, dtype=torch.int64)
    pad = torch.arange(L).unsqueeze(0) >= lens.unsqueeze(1)
    hi[pad] = 0
    hc[pad] = 0
    mask[pad] = int(-1e9)
    ti = torch.randint(1, 63001, (B,), generator=g)
    tc = torch.randint(1, 801, (B,), generator=g)
    label = (torch.rand(B, generator=g) < 0.5).float()
    batch = [t.to(dev) for t in (hi, hc, ti, tc, label, mask, ti.unsqueeze(1).repeat(1, L),
                                 tc.unsqueeze(1).repeat(1, L))]

    def step(i):     # N independent replicas: the path does not shard (DESIGN.md), no collective
        opt.clear_grad()
        loss, _, _ = dm.train_forward(model, None, batch, cfg)
        loss.backward()
        opt.step()
    ms = timed(step, a.iters, 2, world, dev)
    flop = 3 * 2.0 * B * L * (2 * 128 * 80 + 80 * 40 + 40)
    emit(rank, {"config": 4, "what": "DIN AmazonElec-shape train step (7 gathers, fused attention "
                "fwd + bwd, output MLP on the wgmma Linears, SGD)", "n_gpus": world, "B_per_gpu": B,
                "L": L, "ms_per_step": ms, "samples_per_s": B * world / ms * 1e3, "scaling": "weak",
                "parallelism": "replicas only (tables are 63001 x 64: nothing to shard, no collective)",
                "attention_tflops_fp32_lower_bound": round(flop / (ms / 1e3) / 1e12, 2)})


def run_gather(a, rank, world, dev):
    from paddlerec_b200 import ops, sharded
    B, F = a.B, 26
    free, total = torch.cuda.mem_get_info()
    for V in [int(float(v)) for v in a.vocabs.split(",")]:
        for D in [int(d) for d in a.dims.split(",")]:
            rows_local = sharded.shard_rows(V, rank, world)
            need = rows_local * D * 4 + 8 * B * F * (8 + 4 * D)
            fits = torch.tensor([1 if need < 0.85 * free else 0], device=dev)
            if world > 1:
                dist.all_reduce(fits, op=dist.ReduceOp.MIN)
            if not int(fits):
                emit(rank, {"config": 5, "V": V, "D": D, "n_gpus": world, "skipped":
                            "shard of %.0f GB does not fit %.0f GB free per GPU" % (need / 1e9, free / 1e9)})
                continue
            W = torch.empty(max(rows_local, 1), D, device=dev)
            W.uniform_(-0.05, 0.05)
            g = torch.Generator().manual_seed(12345 + rank)
            idl = [torch.randint(0, V, (B, F), generator=g).to(dev) for _ in range(4)]
            if world == 1:
                fn = lambda i: ops.raw_gather(W, idl[i % 4], -1)          # noqa: E731
            else:
                ex = sharded.ShardExchange(V, rank, world)
                ex.prefetch(idl[0])
                ex.finish_prefetch()

                def fn(i):
                    plan = ex.plan(idl[i % 4])            # bucketing + id exchange were prefetched
                    ex.prefetch(idl[(i + 1) % 4])
                    rows = ex.pull(plan, W, -1)
                    out = ops.raw_gather(rows, plan.perm, -1)             # back to position order
                    ex.finish_prefetch()
                    return out
            ms = timed(fn, a.iters, 3, world, dev)
            alg = B * F * (8 + 2 * 4 * D)
            emit(rank, {"config": 5, "what": "Wide&Deep lookup [B,26] -> [B,26,D]" +
                        ("" if world == 1 else " through the row-sharded exchange"), "V": V, "D": D,
                        "n_gpus": world, "B_per_gpu": B, "ms": ms,
                        "gather_GBps_all_gpus": alg * world / ms / 1e6,
                        "gather_GBps_per_gpu": alg / ms / 1e6,
                        "lookups_per_s": B * F * world / ms * 1e3,
                        "table_GB_total": V * D * 4 / 1e9})
            del W
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--what", required=True, choices=["dcn", "din", "gather"])
    ap.add_argument("--B", type=int, default=65536)
    ap.add_argument("--V", type=int, default=100_000_000)
    ap.add_argument("--D", type=int, default=40)
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--iters", type=int, default=8)
    ap.add_argument("--vocabs", default="1e6,1e7,1e8,1e9")
    ap.add_argument("--dims", default="16,64,128")
    a = ap.parse_args()
    rank, world, dev = setup()
    try:
        {"dcn": run_dcn, "din": run_din, "gather": run_gather}[a.what](a, rank, world, dev)
    finally:
        if world > 1:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()
