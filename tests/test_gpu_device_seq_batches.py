"""GPU: SASRec training batches built on the device (runner.fit_on_device with --device_batches): the history collate
kernel (b2r_collate_history) against the host feed dicts, its out-of-range accounting, a device epoch against the same
batches fed by hand, the fixed padded width against the batch maximum, the graphed device route against the eager one,
and the unchanged main.py driving it through the overlay."""
import argparse
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
REF = os.path.join(ROOT, "oracle", "_ref", "src")

pytestmark = [pytest.mark.gpu]


def _corpus():
    sys.path.insert(0, GOLDEN)
    import fit_corpus
    return fit_corpus.build()


def _host_set(corpus, H, neg):
    from rechorus_b200 import plugin
    ds = plugin.SequentialModel.Dataset(types.SimpleNamespace(history_max=H, test_all=0, buffer=1), corpus, "train")
    ds.data["neg_items"] = neg
    return ds


@pytest.mark.parametrize("H", [8, 0])
def test_collate_equals_host_feed_dicts_bit_for_bit(H):
    """collate_general + collate_history vs SequentialModel.Dataset._get_feed_dict + collate_batch (BaseModel.py:236-245,
    135-152) on the same negatives, the host histories right-padded with 0 to Lp; nothing is written beyond row Bn"""
    from rechorus_b200 import ops
    corpus = _corpus()
    dev = torch.device("cuda", 0)
    K, B = 4, 48
    probe = _host_set(corpus, H, None)
    N = len(probe)
    neg = np.random.RandomState(5).randint(1, corpus.n_items, (N, K)).astype(np.int64)
    ds = _host_set(corpus, H, neg)
    his = ops.DeviceHistory(corpus.user_his, corpus.n_users, ds.data["user_id"], ds.data["position"], H, dev)
    Lp = his.width
    assert Lp == (min(H, max(ds.data["position"])) if H > 0 else max(ds.data["position"]))
    users = torch.tensor(np.asarray(ds.data["user_id"], dtype=np.int64), device=dev)
    items = torch.tensor(np.asarray(ds.data["item_id"], dtype=np.int64), device=dev)
    neg_d = torch.from_numpy(neg).to(dev)
    last = ((N - 1) // B) * B
    assert N - last < B                                                   # a ragged last batch exists
    for perm in (None, torch.randperm(N, generator=torch.Generator().manual_seed(9)).to(dev)):
        for start in (0, 2 * B, last):
            Bn = min(B, N - start)
            ou = torch.full((B,), -1, dtype=torch.int64, device=dev)
            oi = torch.full((B, K + 1), -1, dtype=torch.int64, device=dev)
            oh = torch.full((B, Lp), -1, dtype=torch.int64, device=dev)
            ol = torch.full((B,), -1, dtype=torch.int64, device=dev)
            ops.collate_general(users, items, neg_d, perm, start, Bn, ou, oi)
            his.collate(users, perm, start, Bn, oh, ol)
            rows = range(start, start + Bn) if perm is None else perm[start:start + Bn].tolist()
            want = ds.collate_batch([ds._get_feed_dict(int(r)) for r in rows])
            hist = want["history_items"]
            assert hist.shape[1] <= Lp
            assert torch.equal(ou[:Bn].cpu(), want["user_id"])
            assert torch.equal(oi[:Bn].cpu(), want["item_id"])
            assert torch.equal(ol[:Bn].cpu(), want["lengths"])
            assert torch.equal(oh[:Bn].cpu(), F.pad(hist, (0, Lp - hist.shape[1])))
            for t in (ou, oi, oh, ol):
                assert bool((t[Bn:] == -1).all())
    ops.check_ids()


def test_out_of_range_rows_are_clamped_and_counted():
    """rows the setup check would refuse, planted on the device behind it: the kernel clamps them inside the CSR, and the
    next poll raises IndexError"""
    from rechorus_b200 import ops
    corpus = _corpus()
    dev = torch.device("cuda", 0)
    ds = _host_set(corpus, 8, None)
    his = ops.DeviceHistory(corpus.user_his, corpus.n_users, ds.data["user_id"], ds.data["position"], 8, dev)
    users = torch.tensor(np.asarray(ds.data["user_id"], dtype=np.int64), device=dev)
    ops.check_ids()
    users[1] = corpus.n_users + 5                                         # user out of range
    his.positions[2] = 10_000                                             # beyond the user's history
    his.positions[3] = 0                                                  # p < 1
    B = 8
    oh = torch.empty((B, his.width), dtype=torch.int64, device=dev)
    ol = torch.empty(B, dtype=torch.int64, device=dev)
    his.collate(users, None, 0, B, oh, ol)
    torch.cuda.synchronize()
    assert int(ol[3]) == 0 and bool((oh[3] == 0).all())
    assert 0 <= int(ol.min()) and int(ol.max()) <= his.width
    u2 = int(users[2])
    assert int(ol[2]) == min(8, len(corpus.user_his[u2]))
    with pytest.raises(IndexError):
        ops.check_ids()
    ops.check_ids()                                                       # the raise reset the counter


def _runner_args(model_name, flags):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, model_name)
    p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(flags)
    a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_dsb.pt", ""
    return cls, a


SASREC = ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "8", "--num_neg", "5"]


def test_sasrec_device_epoch_equals_the_same_batches_fed_by_hand():
    from rechorus_b200 import ops
    from rechorus_b200.optim import RowSparseOptimizer
    from rechorus_b200.runner import BaseRunner
    flags = SASREC + ["--batch_size", "64", "--num_workers", "0", "--lr", "0.05", "--optimizer", "SGD", "--table_mode",
                      "fused", "--fused_optimizer", "1", "--device_batches", "77"]

    def build():
        cls, a = _runner_args("SASRec", flags)
        corpus = _corpus()
        torch.manual_seed(1)
        model = cls(a, corpus).to(a.device)
        return corpus, model, cls.Dataset(model, corpus, "train"), BaseRunner(a)

    corpus, model, train, runner = build()
    l1 = runner.fit(train, epoch=1)                                       # routed to fit_on_device by the flag
    st = train.__dict__["_b2r_dev"]
    N, K, B, Lp = st["users"].numel(), 5, 64, st["history"].width
    assert Lp == 8
    neg = st["sampler"].sample(st["users"], K, 1)                         # same (seed, epoch) -> same draw
    gen = torch.Generator(device="cuda")
    gen.manual_seed(st["seed"] * 1_000_003 + 1)
    perm = torch.randperm(N, device="cuda", generator=gen)
    # the same epoch by hand on a fresh, identically initialised model, histories from the host feed dicts
    _, model2, train2, _ = build()
    train2.data["neg_items"] = neg.cpu().numpy()
    model2.optimizer = RowSparseOptimizer(model2, "SGD", lr=0.05, l2=0.0)
    model2.set_table_mode("fused")
    model2.train()
    losses = []
    for k in range((N + B - 1) // B):
        rows = perm[k * B:(k + 1) * B]
        host = train2.collate_batch([train2._get_feed_dict(int(r)) for r in rows.tolist()])
        feed = {"user_id": host["user_id"].cuda(), "item_id": host["item_id"].cuda(), "lengths": host["lengths"].cuda(),
                "history_items": F.pad(host["history_items"], (0, Lp - host["history_items"].shape[1])).cuda(),
                "batch_size": rows.numel(), "phase": "train"}
        model2.optimizer.zero_grad()
        ls = model2.loss(model2(feed))
        ls.backward()
        model2.optimizer.step()
        losses.append(ls.detach())
    assert abs(float(torch.stack(losses).mean()) - l1) <= 1e-6
    for (k, pa), (_, pb) in zip(model.named_parameters(), model2.named_parameters()):
        assert torch.equal(pa, pb), k
    l2 = runner.fit(train, epoch=2)
    assert st["epoch"] == 2 and np.isfinite(l2) and abs(l2 - l1) > 0
    gen.manual_seed(st["seed"] * 1_000_003 + 2)
    assert not torch.equal(torch.randperm(N, device="cuda", generator=gen), perm)          # a fresh order ...
    assert not torch.equal(st["sampler"].sample(st["users"], K, 2), neg)                   # ... and fresh negatives
    ops.check_ids()


def test_fixed_width_padding_equals_batch_max_padding():
    """one step on a device batch padded to Lp and on the same batch trimmed to its own maximum length"""
    from rechorus_b200 import ops
    corpus = _corpus()
    dev = torch.device("cuda", 0)
    cls, a = _runner_args("SASRec", ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "50",
                                     "--num_neg", "5", "--table_mode", "dense"])
    torch.manual_seed(4)
    model = cls(a, corpus).to(dev)
    model.train()
    ds = cls.Dataset(model, corpus, "train")
    his = ops.DeviceHistory(corpus.user_his, corpus.n_users, ds.data["user_id"], ds.data["position"], 50, dev)
    users = torch.tensor(np.asarray(ds.data["user_id"], dtype=np.int64), device=dev)
    N, B, K = users.numel(), 64, 5
    perm = torch.from_numpy(np.argsort(np.asarray(ds.data["position"]), kind="stable")).to(dev)   # the shortest first
    items = torch.tensor(np.asarray(ds.data["item_id"], dtype=np.int64), device=dev)
    neg = torch.randint(1, corpus.n_items, (N, K), generator=torch.Generator().manual_seed(2)).to(dev)
    feed = {"user_id": torch.empty(B, dtype=torch.int64, device=dev),
            "item_id": torch.empty((B, K + 1), dtype=torch.int64, device=dev),
            "history_items": torch.empty((B, his.width), dtype=torch.int64, device=dev),
            "lengths": torch.empty(B, dtype=torch.int64, device=dev), "batch_size": B, "phase": "train"}
    ops.collate_general(users, items, neg, perm, 0, B, feed["user_id"], feed["item_id"])
    his.collate(users, perm, 0, B, feed["history_items"], feed["lengths"])
    Lb = int(feed["lengths"].max())
    assert Lb < his.width
    trimmed = dict(feed, history_items=feed["history_items"][:, :Lb].contiguous())

    def step(f):
        for q in model.parameters():
            q.grad = None
        out = model(f)
        loss = model.loss(out)
        loss.backward()
        return out["prediction"].detach().clone(), float(loss.detach()), {k: q.grad.clone() for k, q in model.named_parameters()}

    pa, la, ga = step(feed)
    pb, lb, gb = step(trimmed)
    assert (pa - pb).abs().max() <= 1e-6 and abs(la - lb) <= 1e-6
    for k in ga:
        assert (ga[k] - gb[k]).abs().max() <= 1e-6, k


@pytest.mark.parametrize("model_name,flags", [
    ("SASRec", SASREC + ["--dropout", "0"]),
    ("SASRec", SASREC + ["--dropout", "0.2"]),
    ("NeuMF", ["--emb_size", "32", "--layers", "[32, 16]", "--num_neg", "5", "--dropout", "0.2"])])
def test_graphed_device_route_equals_eager_device_route(model_name, flags):
    from rechorus_b200 import ops
    from rechorus_b200.runner import BaseRunner

    def run(graph):
        cls, a = _runner_args(model_name, flags + [
            "--batch_size", "64", "--num_workers", "0", "--lr", "1e-3", "--l2", "1e-4", "--optimizer", "Adam",
            "--table_mode", "fused", "--fused_optimizer", "1", "--device_batches", "77", "--graph_step", str(graph)])
        corpus = _corpus()
        torch.manual_seed(1)
        model = cls(a, corpus).to(a.device)
        train = cls.Dataset(model, corpus, "train")
        loss = BaseRunner(a).fit(train, epoch=1)
        torch.cuda.synchronize()
        return model, loss, len(train)

    m0, l0, n = run(0)
    m1, l1, _ = run(1)
    assert "_b2r_graphed_step" in m1.__dict__ and "_b2r_graphed_step" not in m0.__dict__
    assert n % 64 != 0 and n // 64 >= 3                                     # warm-up, replays and a ragged last batch
    assert abs(l0 - l1) <= 1e-6 * max(1.0, abs(l0)), (l0, l1)
    for (k, pa), (_, pb) in zip(m0.named_parameters(), m1.named_parameters()):
        assert (pa - pb).abs().max() <= 1e-6, k
    assert m1.optimizer.t == m0.optimizer.t == (n + 63) // 64
    if m0.dropout > 0:
        assert m1.dropout_rng_state() == m0.dropout_rng_state()
        assert m0.dropout_rng_state()[1] == (n + 63) // 64
    ops.check_ids()


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "main.py")),
                    reason="no unmodified reference staged in oracle/_ref")
def test_overlay_sasrec_with_device_batches(tmp_path):
    from tests import test_gpu_overlay as OV
    tmp = str(tmp_path)
    OV._dataset(tmp)
    flags = ["--num_neg", "2", "--num_layers", "2", "--num_heads", "2", "--history_max", "8", "--table_mode", "fused"]
    la, _, _, out = OV._run(tmp, "seq_a", OV.OVERLAY, "SASRec", flags + ["--device_batches", "77"], "0")
    assert len(la) == 2 and all(np.isfinite(la)), out[-2000:]
    lb, _, _, _ = OV._run(tmp, "seq_b", OV.OVERLAY, "SASRec", flags + ["--device_batches", "77"], "0")
    lc, _, _, _ = OV._run(tmp, "seq_c", OV.OVERLAY, "SASRec", flags + ["--device_batches", "78"], "0")
    assert la == lb and la != lc, (la, lb, lc)
