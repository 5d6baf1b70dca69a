"""GPU: the runner's device routes with --tiled_attention 1 at history_max 300, on a corpus whose histories run past 256:
one --device_batches + --graph_step 1 epoch (dropout 0.2) against the same batches collated on the host and fed by hand,
and one --device_metrics 1 evaluation (also under --test_all 1) against the host predict + evaluate_method route.
Evaluation batches are padded to their own longest history, so one evaluation crosses from the default attention
kernels (short batches) to the tiled ones (long batches)."""
import argparse
import types

import numpy as np
import pandas as pd
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu]
HM = 300
MODEL = ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", str(HM), "--tiled_attention", "1"]


def _corpus():
    """4 users with about 350 interactions each and 6 with a handful; the evaluation rows are 8 long histories followed
    by 8 short ones.  Attribute names as in tests/golden/fit_corpus.py."""
    rng = np.random.RandomState(20261017)
    n_users, n_items = 11, 1000                 # the heavy users leave most items to draw negatives from
    users = np.concatenate([rng.randint(1, 5, 1400), rng.randint(5, n_users, 40)])
    rng.shuffle(users)
    df = pd.DataFrame({"user_id": users, "item_id": rng.randint(1, n_items, users.size), "time": np.arange(users.size)})
    user_his, position = {}, []
    for u, i, t in zip(df.user_id, df.item_id, df.time):
        h = user_his.setdefault(int(u), [])
        position.append(len(h))
        h.append((int(i), int(t)))
    df["position"] = position
    heavy = df[df.user_id < 5].tail(8)
    light = df[df.user_id >= 5].tail(8)
    ev = pd.concat([heavy, light]).reset_index(drop=True)
    ev["neg_items"] = [list(rng.randint(1, n_items, 19)) for _ in range(len(ev))]
    train = df.drop(index=list(heavy.index) + list(light.index)).reset_index(drop=True)
    clicked = {u: set() for u in range(n_users)}
    for u, i in zip(train.user_id, train.item_id):
        clicked[int(u)].add(int(i))
    residual = {u: set() for u in range(n_users)}
    for u, i in zip(ev.user_id, ev.item_id):
        residual[int(u)].add(int(i))
    return types.SimpleNamespace(n_users=n_users, n_items=n_items, data_df={"train": train, "dev": ev, "test": ev},
                                 train_clicked_set=clicked, residual_clicked_set=residual, user_his=user_his)


def _runner_args(flags):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    p = plugin.SASRec.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(MODEL + flags)
    a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_long_runner.pt", ""
    return plugin.SASRec, a


def test_graphed_device_epoch_equals_host_batches_fed_by_hand():
    from rechorus_b200 import ops
    from rechorus_b200.optim import RowSparseOptimizer
    from rechorus_b200.runner import BaseRunner
    flags = ["--num_neg", "5", "--dropout", "0.2", "--batch_size", "64", "--num_workers", "0", "--lr", "1e-3",
             "--l2", "1e-4", "--optimizer", "Adam", "--table_mode", "fused", "--fused_optimizer", "1",
             "--device_batches", "77", "--graph_step", "1"]

    def build():
        cls, a = _runner_args(flags)
        corpus = _corpus()
        torch.manual_seed(1)
        model = cls(a, corpus).to(a.device)
        return corpus, model, cls.Dataset(model, corpus, "train"), BaseRunner(a)

    corpus, model, train, runner = build()
    l1 = runner.fit(train, epoch=1)
    assert "_b2r_graphed_step" in model.__dict__
    st = train.__dict__["_b2r_dev"]
    N, K, B, Lp = st["users"].numel(), 5, 64, st["history"].width
    assert Lp == HM and N // B >= 3 and N % B != 0
    neg = st["sampler"].sample(st["users"], K, 1)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(st["seed"] * 1_000_003 + 1)
    perm = torch.randperm(N, device="cuda", generator=gen)
    _, model2, train2, _ = build()
    train2.data["neg_items"] = neg.cpu().numpy()
    model2.optimizer = RowSparseOptimizer(model2, "Adam", lr=1e-3, l2=1e-4)
    model2.set_table_mode("fused")
    model2.train()
    losses, widths = [], []
    for k in range((N + B - 1) // B):
        rows = perm[k * B:(k + 1) * B]
        host = train2.collate_batch([train2._get_feed_dict(int(r)) for r in rows.tolist()])
        widths.append(int(host["lengths"].max()))
        feed = {"user_id": host["user_id"].cuda(), "item_id": host["item_id"].cuda(), "lengths": host["lengths"].cuda(),
                "history_items": F.pad(host["history_items"], (0, Lp - host["history_items"].shape[1])).cuda(),
                "batch_size": rows.numel(), "phase": "train"}
        model2.optimizer.zero_grad()
        ls = model2.loss(model2(feed))
        ls.backward()
        model2.optimizer.step()
        losses.append(ls.detach())
    assert max(widths) == HM                                     # the epoch trains on histories past 256
    assert abs(float(torch.stack(losses).mean()) - l1) <= 1e-6 * max(1.0, abs(l1))
    for (k, pa), (_, pb) in zip(model.named_parameters(), model2.named_parameters()):
        assert (pa - pb).abs().max() <= 1e-6, k
    assert model.dropout_rng_state() == model2.dropout_rng_state()
    ops.check_ids()


@pytest.mark.parametrize("test_all", [0, 1])
def test_device_metrics_equal_host_route_at_history_300(monkeypatch, test_all):
    from rechorus_b200 import lib as Lb
    from rechorus_b200.runner import BaseRunner, device_eval_batches
    h = Lb.load()
    cls, a = _runner_args(["--num_workers", "0", "--eval_batch_size", "4", "--test_all", str(test_all), "--topk",
                           "1,5,10"])
    corpus = _corpus()
    torch.manual_seed(0)
    model = cls(a, corpus).to(a.device)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(5.0)
    ds = cls.Dataset(model, corpus, "dev")
    ds.prepare()
    model.eval()
    runner = BaseRunner(a)
    widths = [int(f["history_items"].shape[1]) for f, _ in device_eval_batches(ds, runner.eval_batch_size)]
    assert max(widths) == HM and min(widths) <= 128              # both routes in one evaluation
    calls = []
    for n in ("b2r_attention_fwd_tiled", "b2r_attention_fwd_rt", "b2r_attention_last_fwd_tiled",
              "b2r_attention_last_fwd"):
        def wrap(*args, _fn=getattr(h, n), _n=n):
            calls.append(_n)
            return _fn(*args)
        monkeypatch.setattr(h, n, wrap)
    preds = runner.predict(ds)
    host = runner.evaluate_method(preds, [1, 5, 10], ["HR", "NDCG"])
    runner.device_metrics = 1
    dev = runner.evaluate(ds, [1, 5, 10], ["HR", "NDCG"])
    assert {"b2r_attention_fwd_tiled", "b2r_attention_fwd_rt", "b2r_attention_last_fwd_tiled",
            "b2r_attention_last_fwd"} <= set(calls), sorted(set(calls))
    assert set(host) == set(dev)
    for k in host:
        assert abs(host[k] - dev[k]) <= 1e-12, (k, host[k], dev[k])
    want = (preds >= preds[:, 0].reshape(-1, 1)).sum(axis=-1)
    got = np.concatenate([ds.model.eval_ranks(f, clicked=c).cpu().numpy()
                          for f, c in device_eval_batches(ds, runner.eval_batch_size)])
    assert np.array_equal(got, want)
