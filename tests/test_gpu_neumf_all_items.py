"""GPU: NeuMF's test_all scores without the materialised candidate matrix -- ops.neumf_score_rows against NeuMF.forward
bit for bit, the route NeuMF's eval_ranks / recommend take on either side of the envelope, the runner's device metrics,
lists and CSV against the host route, and a 1M-item catalogue."""
import argparse
import os
import types

import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = [pytest.mark.gpu]
DEV = torch.device("cuda", 0)


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _model(n_items, d, layers, n_users=40, scale=20.0, integer=False, seed=0):
    from rechorus_b200 import plugin
    p = plugin.NeuMF.parse_model_args(argparse.ArgumentParser())
    a = p.parse_args(["--emb_size", str(d), "--layers", str(list(layers)), "--test_all", "1"])
    a.device, a.model_path = DEV, ""
    torch.manual_seed(seed)
    m = plugin.NeuMF(a, types.SimpleNamespace(n_users=n_users, n_items=n_items)).to(DEV)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for prm in m.parameters():
            if integer:                                         # exact scores: ties everywhere
                prm.copy_(torch.randint(-2, 3, prm.shape, generator=g).float())
            else:
                prm.mul_(scale)                                 # trained-scale weights
    m.eval()
    return m


def _batch(m, Bn, seed=0):
    g = torch.Generator().manual_seed(seed)
    users = torch.randint(0, m.user_num, (Bn,), generator=g).to(DEV)
    targets = torch.randint(1, m.item_num, (Bn,), generator=g).to(DEV)
    ids = torch.arange(m.item_num, dtype=torch.int64, device=DEV).repeat(Bn, 1)
    ids[:, 0] = targets
    return {"user_id": users, "item_id": ids, "batch_size": Bn, "phase": "test"}


def _score(m, feed, b0, b1):
    from rechorus_b200 import ops
    return ops.neumf_score_rows(m.mf_u_embeddings.weight, m.mf_i_embeddings.weight, m.mlp_u_embeddings.weight,
                                m.mlp_i_embeddings.weight, [(l.weight, l.bias) for l in m.mlp], m.prediction.weight,
                                feed["user_id"], feed["item_id"][:, 0], b0, b1)


def _clicked(m, seed=0):
    from rechorus_b200 import ops
    rng = np.random.RandomState(seed)
    train = {u: set(rng.randint(1, m.item_num, rng.randint(0, 40)).tolist()) for u in range(m.user_num)}
    residual = {u: {int(rng.randint(1, m.item_num))} for u in range(0, m.user_num, 2)}
    return train, residual, ops.ClickedSets(train, residual, m.user_num, DEV)


def _host(pred, feed, train, residual, k):
    """BaseRunner.py:244-251's masking, :63's ranks and main.py:121-126's stable sort, in NumPy"""
    pred = pred.cpu().numpy().copy()
    users, target = feed["user_id"].cpu().numpy(), feed["item_id"][:, 0].cpu().numpy()
    for b, u in enumerate(users):
        for it in train.get(int(u), set()) | residual.get(int(u), set()):
            if 1 <= it < pred.shape[1]:
                pred[b, it] = -np.inf
    ranks = (pred >= pred[:, :1]).sum(axis=1)
    order = np.argsort(-pred, axis=1, kind="stable")[:, :k]
    items = np.where(order == 0, target[:, None], order)
    return ranks, items, np.take_along_axis(pred, order, axis=1)


SHAPES = [(32, [32, 16]), (32, [64, 32]), (64, [64]), (64, [64, 32, 16]),
          (32, [96, 16]), (32, [32, 96, 16]), (64, [64, 48])]          # K = 96 layers; a 48-wide last layer


@pytest.mark.parametrize("d,layers", SHAPES)
@pytest.mark.parametrize("n_items,Bn", [(3001, 7), (20011, 3)])
@pytest.mark.parametrize("integer", [False, True])
def test_score_rows_bitwise_equal_forward(d, layers, n_items, Bn, integer):
    from rechorus_b200 import ops
    m = _model(n_items, d, layers, integer=integer)
    feed = _batch(m, Bn)
    assert (Bn * n_items) % 64 != 0                              # the batch's last tile is ragged
    with torch.no_grad():
        ref = m.forward(feed)["prediction"]
    # whole batch, windows straddling 64-row tiles on both sides, single rows
    for b0, b1 in [(0, Bn), (1, Bn - 1), (Bn - 1, Bn), (0, 1), (1, 2)]:
        got = _score(m, feed, b0, b1)
        assert got.shape == (b1 - b0, n_items)
        assert torch.equal(_bits(got), _bits(ref[b0:b1])), (b0, b1)
    ops.check_ids(DEV)


def _spy(monkeypatch, allowed):
    from rechorus_b200 import ops
    real, calls = ops.neumf_score_rows, []

    def spy(*a, **k):
        assert allowed, "the materialised route was expected"
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(ops, "neumf_score_rows", spy)
    return calls


def _check_route(m, Bn, fused, monkeypatch, k=50):
    from rechorus_b200 import ops
    feed = _batch(m, Bn, seed=3)
    train, residual, clicked = _clicked(m)
    with torch.no_grad():
        pred = m.forward(feed)["prediction"]
    want_ranks, want_items, want_scores = _host(pred, feed, train, residual, k)
    calls = _spy(monkeypatch, fused)
    assert (ops.neumf_all_items_error(m.emb_size, m.layers, Bn, m.item_num) is None) == fused
    ranks = m.eval_ranks(feed, clicked=clicked).cpu().numpy()
    items, scores = m.recommend(feed, k, clicked)
    assert bool(calls) == fused
    assert np.array_equal(ranks, want_ranks)
    assert np.array_equal(items.cpu().numpy(), want_items)
    assert np.array_equal(scores.cpu().numpy().view(np.int32), want_scores.astype(np.float32).view(np.int32))


@pytest.mark.parametrize("n_items,fused", [(4095, False), (4096, True)])
def test_route_starts_at_the_forwards_tensor_core_threshold(n_items, fused, monkeypatch):
    _check_route(_model(n_items, 32, [32, 16]), 1, fused, monkeypatch)


@pytest.mark.parametrize("d,layers", [(128, [10]),               # d outside {32, 64}; layer on the SGEMM
                                      (32, [48, 32]),            # second layer K = 48: the forward's SGEMM
                                      (64, [128]),               # wider than the d = 64 kernel's registers
                                      (32, [128, 128, 128])])    # W tiles beyond one CTA's shared memory
def test_shapes_outside_the_envelope_stay_materialised(d, layers, monkeypatch):
    _check_route(_model(3001, d, layers), 3, False, monkeypatch)


def test_training_mode_and_missing_clicked_sets_stay_materialised(monkeypatch):
    m = _model(3001, 32, [32, 16])
    feed = _batch(m, 3)
    _spy(monkeypatch, False)
    with torch.no_grad():
        pred = m.forward(feed)["prediction"]
    assert torch.equal(m.eval_ranks(feed), torch.from_numpy((pred >= pred[:, :1]).sum(1).cpu().numpy()).to(DEV))
    m.train()
    _, _, clicked = _clicked(m)
    m.eval_ranks(feed, clicked=clicked)


def test_two_calls_give_identical_bits_and_bad_ids_raise():
    from rechorus_b200 import ops
    m = _model(20011, 64, [64, 32, 16])
    feed = _batch(m, 3)
    a, b = _score(m, feed, 0, 3), _score(m, feed, 0, 3)
    assert torch.equal(_bits(a), _bits(b))
    ops.check_ids(DEV)
    for key, bad in (("user_id", m.user_num), ("item_id", m.item_num)):
        f = dict(feed)
        f[key] = feed[key].clone()
        if key == "user_id":
            f[key][1] = bad
        else:
            f[key][1, 0] = bad
        _score(m, f, 0, 3)
        with pytest.raises(IndexError):
            ops.check_ids(DEV)


# ---- runner level ------------------------------------------------------------------------------------------------

def _runner_setup(test_all=1):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    n_users, n_items, rows, n_eval = 60, 2000, 900, 80
    rng = np.random.RandomState(5)
    df = pd.DataFrame({"user_id": rng.randint(1, n_users, rows), "item_id": rng.randint(1, n_items, rows),
                       "time": np.arange(rows)})
    ev = df.iloc[rows - n_eval:].copy().reset_index(drop=True)
    ev["neg_items"] = [list(rng.randint(1, n_items, 19)) for _ in range(len(ev))]
    train = df.iloc[:rows - n_eval].copy().reset_index(drop=True)
    clicked = {u: set() for u in range(n_users)}
    for u, i in zip(train.user_id, train.item_id):
        clicked[int(u)].add(int(i))
    residual = {u: set() for u in range(n_users)}
    for u, i in zip(ev.user_id, ev.item_id):
        residual[int(u)].add(int(i))
    corpus = types.SimpleNamespace(n_users=n_users, n_items=n_items, data_df={"train": train, "dev": ev, "test": ev},
                                   train_clicked_set=clicked, residual_clicked_set=residual)
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    p = plugin.NeuMF.parse_model_args(p)
    a = p.parse_args(["--emb_size", "32", "--layers", "[32, 16]", "--num_workers", "0", "--eval_batch_size", "32",
                      "--test_all", str(test_all), "--topk", "1,5,10"])
    a.device, a.model_path, a.log_file = DEV, "/tmp/_b2r_neumf_all.pt", ""
    torch.manual_seed(0)
    model = plugin.NeuMF(a, corpus).to(DEV)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(20.0)
    ds = plugin.NeuMF.Dataset(model, corpus, "test")
    ds.prepare()
    model.eval()
    return model, ds, BaseRunner(a)


def test_runner_metrics_lists_and_csv_equal_the_host_route(tmp_path, monkeypatch):
    from rechorus_b200 import ops
    from rechorus_b200.runner import device_eval_batches
    model, ds, runner = _runner_setup()
    assert ops.neumf_all_items_error(32, [32, 16], 32, 2000) is None and ops.neumf_all_items_error(32, [32, 16], 16, 2000) is None
    preds = runner.predict(ds)
    host = runner.evaluate_method(preds, [1, 5, 10], ["HR", "NDCG"])
    calls = _spy(monkeypatch, True)
    runner.device_metrics = 1
    dev = runner.evaluate(ds, [1, 5, 10], ["HR", "NDCG"])
    assert calls and set(host) == set(dev)
    for k in host:
        assert abs(host[k] - dev[k]) <= 1e-12, (k, host[k], dev[k])
    ranks = np.concatenate([model.eval_ranks(f, clicked=c).cpu().numpy() for f, c in device_eval_batches(ds, 32)])
    assert np.array_equal(ranks, (preds >= preds[:, :1]).sum(axis=-1))

    k = 100
    users, items, scores = runner.recommend(ds, k)
    ref_items, ref_scores = [], []
    for i in range(len(ds)):
        lst = sorted(zip(ds[i]["item_id"], preds[i]), key=lambda x: x[1], reverse=True)[:k]
        ref_items.append([x[0] for x in lst])
        ref_scores.append([x[1] for x in lst])
    ref_items, ref_scores = np.array(ref_items, dtype=np.int64), np.array(ref_scores, dtype=np.float32)
    assert users == list(ds.data["user_id"])
    assert np.array_equal(items, ref_items) and np.array_equal(scores.view(np.int32), ref_scores.view(np.int32))

    rec_df = pd.DataFrame(columns=["user_id", "rec_items", "rec_predictions"])
    rec_df["user_id"] = [ds[i]["user_id"] for i in range(len(ds))]
    rec_df["rec_items"] = [list(r) for r in ref_items]
    rec_df["rec_predictions"] = [list(r) for r in ref_scores]
    ref_path, path = str(tmp_path / "ref.csv"), str(tmp_path / "out" / "rec.csv")
    rec_df.to_csv(ref_path, sep="\t", index=False)
    runner.save_rec_results(ds, path, k, sep="\t")
    assert open(path, "rb").read() == open(ref_path, "rb").read()


# ---- scale -------------------------------------------------------------------------------------------------------

def test_one_million_items():
    from rechorus_b200 import ops
    n_items, d, layers, Bn, k = 1_000_000, 64, [64, 32, 16], 256, 100
    m = _model(n_items, d, layers, n_users=1000)
    feed = _batch(m, Bn, seed=9)
    train, residual, clicked = _clicked(m)
    assert ops.neumf_all_items_error(d, layers, Bn, n_items) is None
    rows = ops.neumf_window_rows(Bn, n_items)
    assert rows * n_items * 4 <= 32 << 20 and rows >= 1
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ranks = m.eval_ranks(feed, clicked=clicked)
    items, scores = m.recommend(feed, k, clicked)
    torch.cuda.synchronize()
    grown = torch.cuda.max_memory_allocated() - base
    assert grown <= rows * n_items * 4 + (8 << 20) + Bn * k * 64, grown
    assert ranks.shape == (Bn,) and items.shape == (Bn, k) and scores.shape == (Bn, k)
    ranks, items, scores = ranks.cpu().numpy(), items.cpu().numpy(), scores.cpu().numpy()
    assert (ranks >= 1).all() and (ranks <= n_items).all() and np.isfinite(scores).all()
    assert (np.diff(scores, axis=1) <= 0).all()
    # sampled rows: the same bits as the forward on that row alone (n_items % 64 == 0, so its tiles are the batch's)
    for b in (0, 77, 255):
        one = {"user_id": feed["user_id"][b:b + 1], "item_id": feed["item_id"][b:b + 1], "batch_size": 1}
        with torch.no_grad():
            ref = m.forward(one)["prediction"]
        assert torch.equal(_bits(_score(m, feed, b, b + 1)), _bits(ref)), b
        r, it, sc = _host(ref, one, train, residual, k)
        assert ranks[b] == r[0] and np.array_equal(items[b], it[0])
        assert np.array_equal(scores[b].view(np.int32), sc[0].astype(np.float32).view(np.int32))
    ops.check_ids(DEV)
