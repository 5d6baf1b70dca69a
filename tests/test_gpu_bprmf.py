"""GPU parity tests: BPRMF scoring / loss / backward / optimizer through the C ABI vs the oracle and vs the
golden fixtures the reference itself produced.  Tolerance (north_star): scores and grads within 1e-5 fp32,
ranks bit-exact."""
import argparse
import types

import numpy as np
import pytest
import torch

from oracle import rechorus_oracle as O
from tests import golden_util as G

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _dev():
    return torch.device("cuda", 0)


def _model(meta, weights, mode="dense"):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    p = argparse.ArgumentParser()
    p = BaseRunner.parse_runner_args(p)
    p = plugin.BPRMF.parse_model_args(p)
    a = p.parse_args(["--emb_size", str(meta["d"]), "--table_mode", mode])
    a.device, a.model_path = _dev(), "/tmp/_b2r_unused.pt"
    m = plugin.BPRMF(a, types.SimpleNamespace(n_users=meta["n_users"], n_items=meta["n_items"])).to(_dev())
    m.load_state_dict(weights)
    m.set_table_mode(mode)
    return m


def _cuda_batch(batch, B):
    out = {k: v.to(_dev()) for k, v in batch.items()}
    out["batch_size"], out["phase"] = B, "train"
    return out


@pytest.mark.parametrize("fixture", G.MODEL_FIXTURES["BPRMF"])
def test_forward_loss_backward_match_reference_fixture(fixture):
    from rechorus_b200 import ops
    meta, w, batch, pred_ref, loss_ref, g_ref = G.load(fixture)
    m = _model(meta, w)
    m.train()
    out = m(_cuda_batch(batch, meta["B"]))
    loss = m.loss(out)
    loss.backward()
    ops.check_ids()
    pred = out["prediction"].detach().cpu()
    assert pred.shape == pred_ref.shape
    assert (pred - pred_ref).abs().max() <= TOL
    assert abs(float(loss) - loss_ref) <= TOL
    assert np.array_equal(O.gt_rank(pred.numpy()), O.gt_rank(pred_ref.numpy()))        # ranks bit-exact
    for k, p in m.named_parameters():
        assert (p.grad.cpu() - g_ref[k]).abs().max() <= TOL, k


@pytest.mark.parametrize("fixture", ["bprmf_k9_trained", "bprmf_d20"])
def test_sparse_and_dense_gradient_forms_agree_bitwise(fixture):
    meta, w, batch, *_ = G.load(fixture)
    grads = {}
    for mode in ("dense", "sparse"):
        m = _model(meta, w, mode)
        m.loss(m(_cuda_batch(batch, meta["B"]))).backward()
        grads[mode] = {k: (p.grad.to_dense() if p.grad.is_sparse else p.grad).cpu() for k, p in m.named_parameters()}
        if mode == "sparse":
            gi = m.i_embeddings.weight.grad
            assert gi.is_sparse
            idx = gi._indices()[0].cpu().numpy()            # as produced: already sorted and unique
            assert np.array_equal(idx, np.unique(batch["item_id"].numpy()))             # sorted unique rows
    for k in grads["dense"]:
        assert torch.equal(grads["dense"][k], grads["sparse"][k]), k


def test_backward_is_bit_reproducible_with_heavy_duplicates():
    torch.manual_seed(0)
    meta = dict(n_users=50, n_items=7, d=64)                     # 7 items -> every row has ~hundreds of writers
    w = O.bprmf_init(50, 7, 64, torch.Generator().manual_seed(1))
    w = {k: v * 30 for k, v in w.items()}
    batch = {"user_id": torch.randint(1, 50, (64,)), "item_id": torch.randint(0, 7, (64, 40))}
    runs = []
    for _ in range(3):
        m = _model(meta, w)
        m.loss(m(_cuda_batch(batch, 64))).backward()
        runs.append(m.i_embeddings.weight.grad.clone())
    assert torch.equal(runs[0], runs[1]) and torch.equal(runs[0], runs[2])
    _, _, g = O.loss_and_grads("BPRMF", w, batch)
    assert (runs[0].cpu() - g["i_embeddings.weight"]).abs().max() <= TOL


def test_out_of_range_ids_are_clamped_and_reported():
    from rechorus_b200 import ops
    U, I = torch.randn(4, 64).cuda(), torch.randn(6, 64).cuda()
    uid = torch.tensor([1, 2]).cuda()
    iid = torch.tensor([[1, 99], [-3, 2]]).cuda()
    pred = ops.rowdot(U, uid, I, iid)
    assert torch.isfinite(pred).all()
    with pytest.raises(IndexError):
        ops.check_ids()
    ops.check_ids()                                   # counter was reset


def test_index_plan_properties():
    from rechorus_b200 import ops
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(0, 1000, (5000,), generator=g)
    plan = ops.IndexPlan(ids.cuda(), 1000)
    nu = plan.count()
    key = plan.sorted_key.cpu().numpy().astype(np.int64)
    pos = plan.sorted_pos.cpu().numpy().astype(np.int64)
    seg = plan.seg_start.cpu().numpy()[:nu]
    uniq = np.unique(ids.numpy())
    assert nu == len(uniq)
    assert np.all(np.diff(key) >= 0) and np.array_equal(np.sort(pos), np.arange(5000))      # sorted, permutation
    assert np.array_equal(ids.numpy()[pos], key)                                             # pairs intact
    assert np.array_equal(key[seg], uniq) and seg[0] == 0
    for a, b in zip(seg, list(seg[1:]) + [5000]):                                             # stable within a run
        assert np.all(np.diff(pos[a:b]) > 0)


@pytest.mark.parametrize("name", ["SGD", "Adam", "Adagrad"])
def test_dense_optimizer_kernel_matches_torch_optim(name):
    from rechorus_b200 import lib as L, ops
    torch.manual_seed(3)
    W0 = torch.randn(37, 21)      # 777 elements: exercises the numel % 4 tail
    Wt = W0.clone().requires_grad_(True)
    topt = getattr(torch.optim, name)([Wt], lr=0.01, weight_decay=1e-3)
    W = W0.clone().cuda()
    m = torch.zeros_like(W) if name == "Adam" else None
    v = torch.zeros_like(W) if name != "SGD" else None
    eps = {"SGD": 0.0, "Adam": 1e-8, "Adagrad": 1e-10}[name]
    for t in range(1, 4):
        grad = torch.randn(37, 21)
        Wt.grad = grad.clone()
        topt.step()
        opt = L.Optim({"SGD": 0, "Adam": 1, "Adagrad": 2}[name], 0.01, 0.9, 0.999, eps, 1e-3,
                      1 - 0.9 ** t, 1 - 0.999 ** t)
        ops.dense_optim(W, grad.cuda(), m, v, opt)
        assert (W.cpu() - Wt.detach()).abs().max() <= 1e-6


@pytest.mark.parametrize("name", ["SGD", "Adam", "Adagrad"])
def test_fused_row_sparse_optimizer_equals_lazy_reference_update(name):
    """Touched rows move exactly as torch.optim would move them given the oracle's gradient; untouched rows
    (and their moments) stay put -- the documented lazy semantics."""
    from rechorus_b200.optim import RowSparseOptimizer
    meta, w, batch, *_ = G.load("bprmf_k9_trained")
    m = _model(meta, w, "fused")
    # a large eps keeps g / (|g| + eps) well-conditioned where gradient entries are ~0 (with the default 1e-8
    # a 1e-9 difference in g moves the update by percents, for torch.optim just as for this kernel)
    eps = {"SGD": 0.0, "Adam": 1e-3, "Adagrad": 1e-3}[name]
    opt = RowSparseOptimizer(m, name, lr=0.05, l2=1e-4, eps=eps)
    cpu_w = {k: v.clone() for k, v in w.items()}
    cpu_state = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in w.items()}
    for t in range(1, 4):
        opt.zero_grad()
        m.loss(m(_cuda_batch(batch, meta["B"]))).backward()
        assert all(p.grad is None for p in m.parameters())          # nothing dense was materialised
        opt.step()
        _, _, g = O.loss_and_grads("BPRMF", cpu_w, batch)
        for k in cpu_w:
            touched = torch.zeros(cpu_w[k].shape[0], dtype=torch.bool)
            touched[batch["user_id" if k.startswith("u_") else "item_id"].reshape(-1)] = True
            W, (M, V) = cpu_w[k], cpu_state[k]
            gr = g[k] + 1e-4 * W
            if name == "SGD":
                Wn = W - 0.05 * gr
            elif name == "Adam":
                Mn, Vn = 0.9 * M + 0.1 * gr, 0.999 * V + 0.001 * gr * gr
                Wn = W - (0.05 / (1 - 0.9 ** t)) * Mn / (Vn.sqrt() / (1 - 0.999 ** t) ** 0.5 + eps)
                M[touched], V[touched] = Mn[touched], Vn[touched]
            else:
                Vn = V + gr * gr
                Wn = W - 0.05 * gr / (Vn.sqrt() + eps)
                V[touched] = Vn[touched]
            W[touched] = Wn[touched]
        for k, p in m.named_parameters():
            assert (p.detach().cpu() - cpu_w[k]).abs().max() <= 2e-6, (name, t, k)


def test_full_size_config2_properties():
    """BASELINE config 2 shapes (1 M items, d=64, B=4096, K=99): size-independent properties + a torch fp32
    check on the same device."""
    from rechorus_b200 import ops
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(2)
    n_items, n_users, B, C, d = 1_000_000, 1_000_000, 4096, 100, 64
    U = torch.randn(n_users, d, device=dev, generator=g) * 0.2
    I = torch.randn(n_items, d, device=dev, generator=g) * 0.2
    uid = torch.randint(1, n_users, (B,), device=dev, generator=g)
    iid = torch.randint(1, n_items, (B, C), device=dev, generator=g)
    pred = ops.rowdot(U, uid, I, iid)
    ref = torch.einsum("bd,bcd->bc", U[uid], I[iid])
    assert (pred - ref).abs().max() <= TOL
    # linearity in the query table
    assert (ops.rowdot(U * 2, uid, I, iid) - 2 * pred).abs().max() <= 2 * TOL
    # column permutation equivariance (the runner shuffles candidates, BaseRunner.py:187-191)
    perm = torch.argsort(torch.rand(B, C, device=dev), dim=-1)
    assert torch.equal(ops.rowdot(U, uid, I, torch.gather(iid, 1, perm)), torch.gather(pred, 1, perm))
    loss, gp = ops.bpr_loss_and_grad(pred)
    assert abs(float(loss) - float(O.bpr_loss(ref.cpu()))) <= TOL
    # gradient checksums: sum over rows of dI equals sum_b (sum_c g[b,c]) u_b ; unique rows match torch.unique
    q = ops.gather_rows(U, uid)
    plan = ops.IndexPlan(iid, n_items)
    uniq, rows = plan.reduce_rows(d, [ops.Source(src=q, n=B * C, coef=gp.reshape(-1), div=C)])
    assert torch.equal(uniq, torch.unique(iid))
    want = (gp.sum(1, keepdim=True).double() * q.double()).sum(0)
    assert (rows.double().sum(0) - want).abs().max() <= 1e-6
    dq = ops.rowdot_bwd_query(gp, I, iid)
    assert (dq - torch.einsum("bc,bcd->bd", gp, I[iid])).abs().max() <= TOL
    ops.check_ids()


@pytest.mark.parametrize("fixture", ["bprmf_k9_trained", "bprmf_d128", "bprmf_d20"])
def test_c_side_train_step_equals_autograd_fused_path(fixture):
    """b2r_bprmf_train_step (one C call) must leave the tables bit-identical to forward/loss/backward through
    autograd followed by RowSparseOptimizer.step()."""
    from rechorus_b200.optim import RowSparseOptimizer
    meta, w, batch, _, loss_ref, _ = G.load(fixture)
    feed = _cuda_batch(batch, meta["B"])
    ma, mb = _model(meta, w, "fused"), _model(meta, w, "fused")
    ma.optimizer = RowSparseOptimizer(ma, "Adam", lr=0.01, l2=1e-5, eps=1e-3)
    mb.optimizer = RowSparseOptimizer(mb, "Adam", lr=0.01, l2=1e-5, eps=1e-3)
    for t in range(3):
        ma.optimizer.zero_grad()
        la = ma.loss(ma(feed))
        la.backward()
        ma.optimizer.step()
        lb = mb.train_step(feed)
        assert abs(float(la) - float(lb)) <= 2e-6       # fused kernel: other reduction order, hardware ex2/rcp
        if t == 0:
            assert abs(float(lb) - loss_ref) <= TOL
        for (k, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
            assert (pa - pb).abs().max() <= 5e-6, (t, k)


def test_train_step_with_prefetched_plan_equals_unprefetched():
    from rechorus_b200.optim import RowSparseOptimizer
    meta, w, batch, *_ = G.load("bprmf_k9_trained")
    g = torch.Generator().manual_seed(3)
    feeds = []
    for _ in range(4):
        feeds.append({"user_id": torch.randint(1, meta["n_users"], (12,), generator=g).cuda(),
                      "item_id": torch.randint(1, meta["n_items"], (12, 10), generator=g).cuda(),
                      "batch_size": 12, "phase": "train"})
    ma, mb = _model(meta, w, "fused"), _model(meta, w, "fused")
    ma.optimizer = RowSparseOptimizer(ma, "Adam", lr=0.01, eps=1e-3)
    mb.optimizer = RowSparseOptimizer(mb, "Adam", lr=0.01, eps=1e-3)
    for t in range(4):
        la = ma.train_step(feeds[t])
        lb = mb.train_step(feeds[t], feeds[t + 1] if t + 1 < 4 else None)
        assert float(la) == float(lb)
        for pa, pb in zip(ma.parameters(), mb.parameters()):
            assert torch.equal(pa, pb)


def test_train_step_without_direct_plan_takes_autograd_route(monkeypatch):
    """Batches whose index plans cannot be sized (B*C > 2^30 - 1) train through the autograd nodes and IndexPlan: with
    DirectPlan reported unavailable, train_step must not enter the single-call step and must leave the same tables as
    forward -> loss -> backward -> RowSparseOptimizer.step() on the direct plans."""
    from rechorus_b200 import ops
    from rechorus_b200.optim import RowSparseOptimizer
    meta, w, batch, *_ = G.load("bprmf_k9_trained")
    feed = _cuda_batch(batch, meta["B"])
    ma, mb = _model(meta, w, "fused"), _model(meta, w, "fused")
    ma.optimizer = RowSparseOptimizer(ma, "Adam", lr=0.01, l2=1e-5, eps=1e-3)
    mb.optimizer = RowSparseOptimizer(mb, "Adam", lr=0.01, l2=1e-5, eps=1e-3)
    losses = []
    for _ in range(3):
        ma.optimizer.zero_grad()
        la = ma.loss(ma(feed))
        la.backward()
        ma.optimizer.step()
        losses.append(float(la))

    def no_step(*a, **k):
        raise AssertionError("the single-call step was entered")

    monkeypatch.setattr(ops.DirectPlan, "available", staticmethod(lambda n, n_rows: False))
    monkeypatch.setattr(ops, "bprmf_train_step", no_step)
    for t in range(3):
        lb = mb.train_step(feed)
        assert abs(losses[t] - float(lb)) <= 2e-6
    for (k, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
        assert (pa - pb).abs().max() <= 1e-6, k
