"""CPU, world_size 2 and 4 over gloo: the exchange bookkeeping of rechorus_b200.shard.ShardedBPRMF (bucketing by owner,
fixed-capacity buffers, all-to-all / all-gather / reduce-scatter wiring, un-permutation) with a torch stand-in for
the local kernels, checked against a single-process oracle of the same global step.  The stand-in lives here, in the
tests: the product backend (CudaBackend) has no CPU path."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import rechorus_oracle as O


class CpuStandIn:
    """test double for shard.CudaBackend (plain torch ops)"""

    def gather_rows(self, T, ids):
        return T[ids]

    def pairdot(self, Q, qidx, T, rows):
        out = (Q[qidx.reshape(-1)] * T[rows.reshape(-1).clamp(min=0)]).sum(-1)
        return torch.where(rows.reshape(-1) >= 0, out, torch.zeros_like(out))

    def bpr_loss_and_grad(self, pred):
        p = pred.detach().clone().requires_grad_(True)
        loss = O.bpr_loss(p)
        loss.backward()
        return loss.detach(), p.grad

    def sum_runs(self, out, key, rows, coef, T):
        keep = rows >= 0
        # every key must occupy ONE contiguous run among the valid pairs (what the CUDA kernel relies on)
        k = key[keep]
        change = torch.nonzero(k[1:] != k[:-1]).numel() + 1 if k.numel() else 0
        assert change == torch.unique(k).numel()
        out.index_add_(0, k, coef[keep].unsqueeze(1) * T[rows[keep]])

    def optimizer_rows(self, W, state, ids, src, coef, src_id, opt):
        g = torch.zeros_like(W)
        keep = ids >= 0
        g.index_add_(0, ids[keep], coef[keep].unsqueeze(1) * src[src_id[keep]])
        touched = torch.zeros(W.shape[0], dtype=torch.bool)
        touched[ids[ids >= 0]] = True
        W[touched] -= opt["lr"] * (g[touched] + opt["wd"] * W[touched])          # SGD is enough for the wiring test

    def make_opt(self, name, lr, betas, eps, wd, t):
        assert name == "SGD"
        return {"lr": lr, "wd": wd}


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


N_USERS, N_ITEMS, D, B, C, STEPS, LR = 20, 30, 8, 6, 5, 2, 0.5


def _global_tables():
    g = torch.Generator().manual_seed(11)
    return torch.randn(N_USERS, D, generator=g) * 0.5, torch.randn(N_ITEMS, D, generator=g) * 0.5


def _batches(rank):
    g = torch.Generator().manual_seed(100 + rank)
    return [(torch.randint(0, N_USERS, (B,), generator=g), torch.randint(0, N_ITEMS, (B, C), generator=g))
            for _ in range(STEPS)]


def _worker(rank, world, port, out_q):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from rechorus_b200.shard import ShardedBPRMF
    m = ShardedBPRMF(N_USERS, N_ITEMS, D, torch.device("cpu"), backend=CpuStandIn(), optimizer="SGD", lr=LR,
                     cap_factor=3.0)
    U, I = _global_tables()
    pad = lambda T, rows: torch.cat([T, torch.zeros(rows * world - T.shape[0], D)])   # last shard may be ragged
    m.U.copy_(pad(U, m.rows_u)[rank * m.rows_u:(rank + 1) * m.rows_u])
    m.I.copy_(pad(I, m.rows_i)[rank * m.rows_i:(rank + 1) * m.rows_i])
    losses = []
    for uid, iid in _batches(rank):
        pred, _ = m.scores(uid, iid)
        losses.append(float(m.train_step(uid, iid)))
    # by value (numpy), not as shared-memory tensors: the parent may unpickle after this process has exited
    out_q.put((rank, m.U.numpy().copy(), m.I.numpy().copy(), losses, pred.numpy().copy()))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_step_equals_single_process_oracle(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r, U, I, losses, pred = q.get(timeout=240)
        got[r] = (torch.from_numpy(U), torch.from_numpy(I), losses, torch.from_numpy(pred))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    # single-process replay of the same global steps: objective = mean over the W*B samples
    U, I = _global_tables()
    U, I = U.clone().requires_grad_(True), I.clone().requires_grad_(True)
    per_rank = [_batches(r) for r in range(world)]
    for t in range(STEPS):
        losses = [O.bpr_loss(O.bprmf_scores({"u_embeddings.weight": U, "i_embeddings.weight": I}, *per_rank[r][t]))
                  for r in range(world)]
        for r in range(world):
            assert abs(float(losses[r]) - got[r][2][t]) < 1e-5
        total = sum(losses) / world
        gU, gI = torch.autograd.grad(total, [U, I])
        with torch.no_grad():
            U -= LR * gU
            I -= LR * gI
    rows_u, rows_i = got[0][0].shape[0], got[0][1].shape[0]
    U_sh = torch.cat([got[r][0] for r in range(world)])[:N_USERS]
    I_sh = torch.cat([got[r][1] for r in range(world)])[:N_ITEMS]
    assert rows_u * world >= N_USERS and rows_i * world >= N_ITEMS
    assert (U_sh - U.detach()).abs().max() < 1e-5
    assert (I_sh - I.detach()).abs().max() < 1e-5


def test_bucket_by_owner_is_a_stable_partition():
    from rechorus_b200.shard import _bucket_by_owner
    owner = torch.tensor([2, 0, 1, 2, 0, 0, 1])
    order, owner_sorted, rank, counts = _bucket_by_owner(owner, 4)
    assert order.tolist() == [1, 4, 5, 2, 6, 0, 3] and owner_sorted.tolist() == [0, 0, 0, 1, 1, 2, 2]
    assert rank.tolist() == [0, 1, 2, 0, 1, 0, 1] and counts.tolist() == [3, 2, 2, 0]


def test_exchange_keyword_defaults_to_nccl_off_cuda_and_refuses_p2p_there():
    from rechorus_b200.shard import ShardedBPRMF
    cpu = torch.device("cpu")
    assert ShardedBPRMF(N_USERS, N_ITEMS, D, cpu, backend=CpuStandIn(), optimizer="SGD").exchange == "nccl"
    assert ShardedBPRMF(N_USERS, N_ITEMS, D, cpu, optimizer="SGD", exchange="nccl").exchange == "nccl"
    for kw in ({"backend": CpuStandIn()}, {}):
        with pytest.raises(ValueError, match="p2p"):
            ShardedBPRMF(N_USERS, N_ITEMS, D, cpu, optimizer="SGD", exchange="p2p", **kw)
    with pytest.raises(ValueError, match="exchange"):
        ShardedBPRMF(N_USERS, N_ITEMS, D, cpu, backend=CpuStandIn(), optimizer="SGD", exchange="nvlink")
