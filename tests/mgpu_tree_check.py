"""Device tree fits with one rank per process, run under torchrun (one rank per GPU):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29541 tests/mgpu_tree_check.py

Every rank holds a contiguous row shard (ensemble.row_partition) of the same seeded global dataset and fits on it with
se_tree_fit / se_tree_fit_classifier; each level's histogram is all-reduced across the ranks.  The labels, weights and
bag counts are small dyadic values, so every histogram sum is exact in any order: every rank's tree must equal, bit for
bit, the tree rank 0 fits on the WHOLE data in a context of its own, and the ranks' outputs concatenated must equal
that fit's output."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    import torch.distributed as dist
    from spark_ensemble_b200 import _native as N
    from spark_ensemble_b200.context import Context
    from spark_ensemble_b200.ensemble import row_partition
    from spark_ensemble_b200.learners import DeviceDecisionTreeRegressor
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    ctx = Context(local)
    uid = torch.zeros(N.COMM_ID_BYTES, dtype=torch.uint8, device="cuda")
    if rank == 0:
        uid = torch.frombuffer(bytearray(Context.comm_unique_id()), dtype=torch.uint8).cuda()
    dist.broadcast(uid, 0)
    ctx.comm_init(world, rank, bytes(uid.cpu().numpy().tobytes()))
    assert ctx.comm_info() == (world, rank)

    rng = np.random.default_rng(29)
    n, d, K = 100_003, 7, 5
    X = rng.integers(0, 16, (n, d)).astype(np.float32)
    r = (((X[:, 0] > 7) * 4 + X[:, 1] % 3 + rng.integers(-4, 4, n)) / 4).astype(np.float32)
    y = ((3 * X[:, 0] + X[:, 2] + rng.integers(0, 3, n)) % K).astype(np.float32)
    w = rng.integers(1, 5, n).astype(np.float32)
    bag = rng.integers(0, 3, n).astype(np.float32)
    cands = DeviceDecisionTreeRegressor(maxBins=32, seed=3).split_candidates(X)
    sub = np.array([6, 0, 1, 2, 4], np.int32)

    def load(c, rows):
        m = rows.stop - rows.start
        c.alloc(N.SLOT_X, d, m)
        c.upload_rowmajor(N.SLOT_X, X[rows])
        for slot, v in ((N.SLOT_R, r), (N.SLOT_Y, y), (N.SLOT_W, w), (N.SLOT_BAG, bag)):
            c.alloc(slot, 1, m)
            c.upload(slot, v[rows])
        c.alloc(N.SLOT_H, 1, m)
        c.alloc(N.SLOT_PROBA, K, m)
        c.tree_fit_bins(cands)

    def fits(c, m):
        reg = c.tree_fit(N.SLOT_R, 0, N.SLOT_W, 0, True, subspace=sub, max_depth=6, out_slot=N.SLOT_H)
        reg_out = np.asarray(c.download(N.SLOT_H)).reshape(1, m)
        cls = c.tree_fit_classifier(N.SLOT_Y, K, 0, N.SLOT_W, 0, True, subspace=sub, impurity="entropy", max_depth=5,
                                    proba=True, out_slot=N.SLOT_PROBA)
        cls_out = np.asarray(c.download(N.SLOT_PROBA)).reshape(K, m)
        return [(reg, reg_out), (cls, cls_out)]

    s0, s1 = row_partition(n, world, rank)
    load(ctx, slice(s0, s1))
    mine = fits(ctx, s1 - s0)
    gathered = [None] * world
    dist.all_gather_object(gathered, mine)
    if rank == 0:
        with Context(local) as whole:
            load(whole, slice(0, n))
            ref = fits(whole, n)
        for which, (t_ref, o_ref) in enumerate(ref):
            assert t_ref["feature"].size > 7, which
            for rk in range(world):
                t = gathered[rk][which][0]
                for key in t_ref:
                    np.testing.assert_array_equal(t[key], t_ref[key], err_msg=f"fit {which} rank {rk} {key}")
            out = np.concatenate([gathered[rk][which][1] for rk in range(world)], axis=1)
            np.testing.assert_array_equal(out.view(np.uint32), o_ref.view(np.uint32))
    dist.barrier()
    if rank == 0:
        print(f"MGPU_TREE_OK world={world}")
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
