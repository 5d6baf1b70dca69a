"""CPU: the impression training epoch's batches and row order against what the reference's own ImpressionRunner.fit passes
its model (tests/golden/impression_fit.npz, tests/golden/make_impression_fit_golden.py), and the route decision of the
overlay's B200ImpressionRunner.fit."""
import os
import types

import numpy as np
import pytest
import torch

from tests.impression_oracle import impression_collate, impression_history

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "impression_fit.npz")
TAGS = ("general", "seq")


def impression_labels(pos_num, neg_num, mp: int, mn: int) -> np.ndarray:
    """int64 [B, mp + mn]: ImpressionRunner.fit's labels (helpers/ImpressionRunner.py:186-189) from the raw pos_num /
    neg_num, clipped as _get_feed_dict clips them: 1 / -1 on the positive slots, 0 / -1 on the negative ones"""
    P = np.minimum(np.asarray(pos_num, dtype=np.int64), mp)[:, None]
    Q = np.minimum(np.asarray(neg_num, dtype=np.int64), mn)[:, None]
    return np.concatenate([np.where(np.arange(mp) < P, 1, -1), np.where(np.arange(mn) < Q, 0, -1)], axis=1)


def fixture_rows(z, tag):
    """the training set of one Dataset kind as lists: (rows, users, positions, pos lists, neg lists, user_his pos)"""
    users, position = z["user_id"], z["position"]
    pp, pf, npt, nf = z["pos_ptr"], z["pos_flat"], z["neg_ptr"], z["neg_flat"]
    rows = np.arange(len(users)) if tag == "general" else np.flatnonzero(position > 0)
    hp, hf = z["his_ptr"], z["his_flat"]
    his = {int(u): [(int(x), 0) for x in hf[hp[i]:hp[i + 1]]] for i, u in enumerate(z["his_users"])}
    return (rows, users[rows], position[rows], [list(pf[pp[r]:pp[r + 1]]) for r in rows],
            [list(nf[npt[r]:npt[r + 1]]) for r in rows], his)


def test_fixture_covers_the_edges():
    z = np.load(GOLDEN)
    mp, mn, B = (int(z[k]) for k in ("mp", "mn", "B"))
    assert mn > mp
    for tag in TAGS:
        _, _, _, pos, neg, _ = fixture_rows(z, tag)
        assert len(pos) == int(z[f"{tag}/rows"]) and len(pos) % B != 0
        assert max(len(p) for p in pos) > mp and max(len(n) for n in neg) > mn
    assert sorted(int(z[f"{t}/num_workers"]) for t in TAGS) == [0, 2]


@pytest.mark.parametrize("tag", TAGS)
def test_reference_shuffle_and_collate_reproduce_the_reference_fit(tag):
    from rechorus_b200.runner import reference_shuffle
    z = np.load(GOLDEN)
    mp, mn, B, H = (int(z[k]) for k in ("mp", "mn", "B", "history_max"))
    _, users, position, pos, neg, his = fixture_rows(z, tag)
    N = len(users)
    torch.manual_seed(int(z["seed"]))
    for e in range(1, int(z["epochs"]) + 1):
        order = reference_shuffle(N).numpy()
        for bi, s in enumerate(range(0, N, B)):
            r = order[s:s + B]
            uid, iid = impression_collate([pos[i] for i in r], [neg[i] for i in r], users[r], mp, mn)
            lab = impression_labels([len(pos[i]) for i in r], [len(neg[i]) for i in r], mp, mn)
            assert np.array_equal(uid, z[f"{tag}/{e}/{bi}/user_id"]), (e, bi)
            assert np.array_equal(iid, z[f"{tag}/{e}/{bi}/item_id"]), (e, bi)
            assert np.array_equal(lab, z[f"{tag}/{e}/{bi}/labels"]), (e, bi)
            if tag == "seq":
                hi, ln = impression_history(his, users[r], position[r], H)
                assert np.array_equal(hi, z[f"{tag}/{e}/{bi}/history_items"]), (e, bi)
                assert np.array_equal(ln, z[f"{tag}/{e}/{bi}/lengths"]), (e, bi)
        assert f"{tag}/{e}/{(N + B - 1) // B}/user_id" not in z.files
        assert np.array_equal(torch.get_rng_state().numpy(), z[f"{tag}/{e}/rng"]), e


def test_reference_shuffle_matches_a_dataloader_epoch():
    from torch.utils.data import DataLoader

    from rechorus_b200.runner import reference_shuffle
    torch.manual_seed(5)
    order = reference_shuffle(37)
    after = torch.get_rng_state()
    torch.manual_seed(5)
    got = torch.cat(list(DataLoader(list(range(37)), batch_size=8, shuffle=True, num_workers=0)))
    assert torch.equal(got, order) and torch.equal(after, torch.get_rng_state())


# ---- route decision --------------------------------------------------------------------------------------------------

class _StubImpressionRunner:
    """stands in for the reference's ImpressionRunner: records that its fit ran"""

    @staticmethod
    def parse_runner_args(parser):
        return parser

    def __init__(self, args):
        self.calls = []

    def fit(self, data, epoch=-1):
        self.calls.append(epoch)
        return 0.5


def _setup(monkeypatch, flag=1, pos_num=True, neg_num=True, rows=2, kernels=True):
    from rechorus_b200 import overlay, runner
    device_calls = []
    monkeypatch.setattr(runner, "fit_impression_on_device", lambda r, d, e: device_calls.append(e) or 0.25)
    cls = overlay._make_impression_runner_module(_StubImpressionRunner).B200ImpressionRunner
    run = cls(types.SimpleNamespace(device_batches=flag))
    model = types.SimpleNamespace()
    if kernels:
        model.eval_ranks = lambda *a, **k: None
    data = {"user_id": list(range(rows))}
    if pos_num:
        data["pos_num"] = [1] * rows
    if neg_num:
        data["neg_num"] = [1] * rows
    return run, types.SimpleNamespace(model=model, data=data), device_calls


def test_device_route_taken_when_every_condition_holds(monkeypatch):
    run, ds, dev = _setup(monkeypatch)
    assert run.fit(ds, 3) == 0.25 and dev == [3] and run.calls == []


@pytest.mark.parametrize("case", ["no_flag", "no_pos_num", "no_neg_num", "no_rows", "host_model"])
def test_excluded_cases_keep_the_reference_fit(monkeypatch, case):
    kw = {"no_flag": dict(flag=0), "no_pos_num": dict(pos_num=False), "no_neg_num": dict(neg_num=False),
          "no_rows": dict(rows=0), "host_model": dict(kernels=False)}[case]
    run, ds, dev = _setup(monkeypatch, **kw)
    assert run.fit(ds, 4) == 0.5
    assert run.calls == [4] and dev == []


def test_parser_knows_device_batches():
    import argparse

    from rechorus_b200 import overlay
    cls = overlay._make_impression_runner_module(_StubImpressionRunner).B200ImpressionRunner
    p = cls.parse_runner_args(argparse.ArgumentParser())
    a = p.parse_args(["--device_batches", "1", "--device_metrics", "1"])
    assert a.device_batches == 1 and a.device_metrics == 1
    assert "not a seed" in next(x.help for x in p._actions if x.dest == "device_batches")
