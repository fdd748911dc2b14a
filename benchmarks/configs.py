#!/usr/bin/env python
"""The five BASELINE.json configurations, device-resident.

    python benchmarks/configs.py [--out /tmp/configs_n1.json]                       # one GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \\
        --master-port 29541 benchmarks/configs.py --out /tmp/configs_n8.json         # one rank per GPU

C1 GBMRegressor cpusmall 20 rounds (host base learner: the reference's plumbing case, timed end to end; rank 0 only)
C2 GBMRegressor 10 M x 64 squared, 100 rounds, 1 GPU     (one cooperative launch per round)
C3 GBMClassifier 50 M rows GLOBAL, bernoulli, rows sharded over the ranks: persistent on-device Brent line search
   (cross-GPU sums inside the kernel) + fused update per round
C4 BoostingClassifier SAMME.R 26 classes, 100 M rows GLOBAL sharded: fused error + weight update + Σw' per round
C5 BaggingRegressor.transform 512 models x 50 M rows GLOBAL sharded: aggregation kernel (no collective)
Global sizes are divided by the number of ranks (strong scaling: the configuration BASELINE.json states); times are
the max over ranks.  The direction of every device round is a fixed synthetic vector correlated with the label (the
base learner is third party and not timed).  Every multi-GPU scalar is cross-checked against an independent
torch.distributed all-reduce of the per-rank values (`consistency`)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from spark_ensemble_b200 import _native as N  # noqa: E402
from spark_ensemble_b200.context import Context  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--c3-rounds", type=int, default=50)
    args = ap.parse_args()
    sc = 0.1 if args.quick else 1.0
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    dist = None
    if world > 1:
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    res = {"world": world}

    def allmax(v):
        if dist is None:
            return float(v)
        import torch
        t = torch.tensor([float(v)], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def allsum(v):
        if dist is None:
            return float(v)
        import torch
        t = torch.tensor([float(v)], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.SUM)
        return float(t.item())

    def barrier():
        ctx.sync()
        if dist is not None:
            dist.barrier()

    # ---- C1 (rank 0, single process semantics)
    if rank == 0 and world == 1:
        from spark_ensemble_b200 import DataFrame
        from spark_ensemble_b200.learners import DecisionTreeRegressor
        from spark_ensemble_b200.regression import GBMRegressor
        d = np.load(os.path.join(ROOT, "tests", "golden", "cpusmall.npz"))
        X, y = d["X"].astype(np.float32), d["y"].astype(np.float64)
        t0 = time.perf_counter()
        m = GBMRegressor().setBaseLearner(DecisionTreeRegressor(maxDepth=5)).setNumBaseLearners(20).fit(DataFrame(features=X, label=y))
        dt = time.perf_counter() - t0
        res["C1"] = {"config": "GBMRegressor cpusmall 8192x12, 20 rounds, squared (sklearn tree on host)", "seconds": dt,
                     "final_train_loss": m.trainingHistory[-1]["trainLoss"]}
        print("C1", res["C1"], flush=True)
    ctx = Context(local)
    if world > 1:
        import torch
        uid = torch.zeros(N.COMM_ID_BYTES, dtype=torch.uint8, device="cuda")
        if rank == 0:
            uid = torch.frombuffer(bytearray(Context.comm_unique_id()), dtype=torch.uint8).cuda()
        dist.broadcast(uid, 0)
        ctx.comm_init(world, rank, bytes(uid.cpu().numpy().tobytes()))
        res["p2p_active"] = bool(ctx.comm_p2p_active())
    seed = 1000 * (rank + 1)

    def correlated_direction(loss):
        """H <- y*s + N(0, 0.5) on the device (a base learner correlated with the label); F <- 0."""
        ctx.fill_synthetic(N.SLOT_F, "normal", seed + 3, 0.0, 0.5)
        ctx.copy_slot(N.SLOT_H, N.SLOT_Y)
        ctx.gbm_update([0.5 if loss == "squared" else 1.0], residual=False, loss=False)
        ctx.copy_slot(N.SLOT_H, N.SLOT_F)
        ctx.fill(N.SLOT_F, 0.0)

    # ---- C2 (1 GPU) / C3 (sharded): device rounds through se_gbm_round
    todo = []
    if world == 1:
        todo.append(("C2", "squared", int(10e6 * sc), 100))
    todo.append(("C3", "bernoulli", int(50e6 * sc) // world // 4 * 4, args.c3_rounds))
    for name, loss, n, rounds in todo:
        ctx.gbm_configure(n, 0, 1, loss, 0.0, False)
        ctx.fill_synthetic(N.SLOT_Y, "bernoulli" if loss == "bernoulli" else "normal", seed + 1, 0.4, 1.0)
        correlated_direction(loss)
        ctx.gbm_pseudo_residuals(False)
        for _ in range(3):
            ctx.gbm_round(0.1, True, 1e-6, 100, residual=True)
        barrier()
        evals = 0
        t0 = time.perf_counter()
        for _ in range(rounds):
            a, ls, ne = ctx.gbm_round(0.1, True, 1e-6, 100, residual=True)
            evals += ne
        ctx.sync()
        dt = allmax(time.perf_counter() - t0)
        # consistency: the train loss the library returned (summed across GPUs inside its kernels) vs an
        # independent all-reduce of per-rank local losses (a single-GPU context over the same shard)
        res[name] = {"config": f"{loss} {n * world} rows global ({n} per GPU x {world}), {rounds} rounds, Brent tol 1e-6, lr 0.1",
                     "ms_per_round": 1e3 * dt / rounds, "rows_per_s": n * world * rounds / dt, "brent_evals_per_round": evals / rounds,
                     "one_launch_round": int(ctx.get_option("last_round_fused")),
                     "line_search": "n/a (squared: in the round kernel)" if loss == "squared" else
                     {0: "one launch per evaluation", 1: "one persistent launch (device Brent)", 2: "host Brent"}[int(ctx.get_option("ls_mode"))],
                     "last_alpha": a}
        if world > 1:
            # every rank must hold the same alpha bit for bit
            import torch
            t = torch.tensor([a], dtype=torch.float64, device="cuda")
            tl = [torch.zeros_like(t) for _ in range(world)]
            dist.all_gather(tl, t)
            res[name]["alpha_identical_on_all_ranks"] = bool(all(float(x) == a for x in tl))
        if rank == 0:
            print(name, res[name], flush=True)
    for s in (N.SLOT_F, N.SLOT_H, N.SLOT_R):
        ctx.free(s)
    # ---- C4
    K, n, rounds = 26, int(100e6 * sc) // world // 4 * 4, 20
    ctx.boost_configure(n, K, True)
    ctx.fill_synthetic(N.SLOT_Y, "randint", seed + 1, 0, K)
    ctx.fill_synthetic(N.SLOT_PROBA, "uniform", seed + 2, 0.001, 0.08)
    ctx.fill(N.SLOT_BW, 1.0)
    sw = ctx.slot_sum(N.SLOT_BW)
    assert sw == float(n * world), (sw, n * world)   # GLOBAL sum (in-kernel cross-GPU exchange)
    for _ in range(2):
        e, sw = ctx.boost_real_update(sw)
    barrier()
    t0 = time.perf_counter()
    for _ in range(rounds):
        e, sw = ctx.boost_real_update(sw)
    ctx.sync()
    dt = allmax(time.perf_counter() - t0)
    # consistency: global Σw' from the kernel's peer exchange vs NCCL all-reduce of the per-rank sums of the weights
    local_sum = float(np.sum(ctx.download(N.SLOT_BW).astype(np.float64)))
    sw_check = allsum(local_sum)
    res["C4"] = {"config": f"SAMME.R K={K}, {n * world} rows global ({n} per GPU x {world}), {rounds} rounds",
                 "ms_per_round": 1e3 * dt / rounds, "rows_per_s": n * world * rounds / dt,
                 "gbs_per_gpu": (4 * K + 12) * n * rounds / dt / 1e9,
                 "consistency": {"sum_w_library": sw, "sum_w_independent_allreduce": sw_check,
                                 "rel_diff": abs(sw - sw_check) / sw_check}}
    assert abs(sw - sw_check) <= 1e-6 * sw_check, res["C4"]
    if rank == 0:
        print("C4", res["C4"], flush=True)
    ctx.free(N.SLOT_PROBA)
    # ---- C5
    M, n, reps = 512, int(50e6 * sc) // world // 4 * 4, 10
    ctx.agg_configure(N.AGG_BAGGING_REGRESSOR, M, 0, 1, 0, n)
    ctx.fill_synthetic(N.SLOT_P, "normal", seed + 7, 0.0, 1.0)
    ctx.agg_run()
    barrier()
    t0 = time.perf_counter()
    for _ in range(reps):
        ctx.agg_run()
    ctx.sync()
    dt = allmax(time.perf_counter() - t0)
    res["C5"] = {"config": f"BaggingRegressor.transform M={M}, {n * world} rows global ({n} per GPU x {world})",
                 "ms_per_pass": 1e3 * dt / reps, "rows_per_s": n * world * reps / dt, "gbs_per_gpu": (4 * M + 4) * n * reps / dt / 1e9}
    if rank == 0:
        print("C5", res["C5"], flush=True)
    ctx.close()
    if rank == 0 and args.out:
        json.dump(res, open(args.out, "w"), indent=1)
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
