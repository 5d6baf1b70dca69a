#!/usr/bin/env python
"""Config-5 style run of the row-sharded BPRMF path under torchrun (one rank per GPU, NCCL):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29511 \
        tools/shard_bench.py --n_items 100000000 --n_users 1000000 --d 128 --B 4096 --K 255 --steps 20 --warmup 5 [--check]

--check: small sizes; every rank verifies scores against a replicated full-table computation (all-gathered shards).
Prints one JSON line on rank 0: user x item / s over all ranks (max-over-ranks CUDA-event time).
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n_items", type=int, default=100_000_000)
    ap.add_argument("--n_users", type=int, default=1_000_000)
    ap.add_argument("--emb", type=int, default=128)
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--K", type=int, default=255)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--optimizer", type=str, default="Adam")
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--exchange", choices=("p2p", "nccl"), default="p2p",
                    help="p2p: kernels store into the peers' symmetric memory; nccl: the collective form")
    ap.add_argument("--torch_profile", action="store_true", help="print a torch.profiler kernel table for 3 steps (rank 0)")
    a = ap.parse_args()
    rank, world, local = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    from rechorus_b200 import ops
    from rechorus_b200.shard import ShardedBPRMF
    m = ShardedBPRMF(a.n_users, a.n_items, a.emb, dev, optimizer=a.optimizer, lr=1e-3, init_std=0.1 if a.check else 0.01,
                     exchange=a.exchange)
    C = a.K + 1
    g = torch.Generator(device=dev).manual_seed(1234 + rank)
    pool = [(torch.randint(1, a.n_users, (a.B,), device=dev, generator=g),
             torch.randint(1, a.n_items, (a.B, C), device=dev, generator=g)) for _ in range(4)]
    if a.check:
        uid, iid = pool[0]
        pred, _ = m.scores(uid, iid)
        if world > 1:
            U = torch.empty(world * m.rows_u, a.emb, device=dev); dist.all_gather_into_tensor(U, m.U)
            I = torch.empty(world * m.rows_i, a.emb, device=dev); dist.all_gather_into_tensor(I, m.I)
        else:
            U, I = m.U, m.I
        ref = torch.einsum("bd,bcd->bc", U[uid], I[iid])
        err = float((pred - ref).abs().max())
        # exact expected SGD step of the global objective (mean over the W*B samples) from the gathered tables
        if world > 1:
            uid_all = torch.empty(world * uid.numel(), dtype=torch.int64, device=dev)
            iid_all = torch.empty(world * iid.numel(), dtype=torch.int64, device=dev)
            dist.all_gather_into_tensor(uid_all, uid)
            dist.all_gather_into_tensor(iid_all, iid.reshape(-1))
            iid_all = iid_all.view(-1, C)
        else:
            uid_all, iid_all = uid, iid
        Ug, Ig = U.clone().requires_grad_(True), I.clone().requires_grad_(True)
        p_all = torch.einsum("bd,bcd->bc", Ug[uid_all], Ig[iid_all])
        pos, neg = p_all[:, :1], p_all[:, 1:]
        wgt = torch.softmax(neg - neg.max(), dim=1)
        total = -torch.log(((pos - neg).sigmoid() * wgt).sum(1).clamp(1e-8, 1 - 1e-8)).mean()
        gU, gI = torch.autograd.grad(total, [Ug, Ig])
        loss = m.train_step(uid, iid)
        lo_i, lo_u = rank * m.rows_i, rank * m.rows_u
        exp_I = (I - 1e-3 * gI)[lo_i:lo_i + m.rows_i]
        exp_U = (U - 1e-3 * gU)[lo_u:lo_u + m.rows_u]
        upd_err = max(float((m.I - exp_I).abs().max()), float((m.U - exp_U).abs().max()))
        # relative to the size of the update itself (lr * |g| is tiny at init): the step must be reproduced, not lost
        upd_rel = float(((m.I - I[lo_i:lo_i + m.rows_i]) - (exp_I - I[lo_i:lo_i + m.rows_i])).abs().max()
                        / (1e-3 * gI.abs().max()).clamp_min(1e-30))
        ok = upd_err <= 1e-6 and upd_rel <= 1e-3
        ops.check_ids(dev)
        print(json.dumps({"rank": rank, "check_max_abs_err": err, "update_max_abs_err": upd_err, "update_rel_err": upd_rel, "update_ok": ok, "loss": float(loss)}), flush=True)
        assert err <= 1e-5 and ok
    for k in range(a.warmup):
        m.train_step(*pool[k % 4])
    torch.cuda.synchronize()
    if a.torch_profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for k in range(3):
                m.train_step(*pool[k % 4])
            torch.cuda.synchronize()
        if rank == 0:
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=25, max_name_column_width=70), flush=True)
    if world > 1:
        dist.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(a.steps):
        loss = m.train_step(*pool[k % 4])
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms.item()) / a.steps
    ops.check_ids(dev)
    if rank == 0:
        print(json.dumps({"metric": "training samples/sec (user x (1+neg))", "value": world * a.B * C / (ms * 1e-3),
                          "unit": "user*item/s", "n_gpus": world, "ms_per_step": ms, "scaling": "weak",
                          "config": {"workload": f"sharded BPRMF d={a.emb} n_items={a.n_items} n_users={a.n_users} "
                                                 f"B={a.B}/GPU K={a.K}", "parallelism": f"row-range shards x{world}, score routing",
                                     "optimizer": a.optimizer + " (row-sparse)"},
                          "loss": float(loss), "mem_GB": torch.cuda.max_memory_allocated() / 1e9}), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
