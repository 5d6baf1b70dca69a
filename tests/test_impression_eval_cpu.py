"""CPU: the impression evaluation's definitions against the reference's own outputs (tests/golden/impression_eval.npz,
tests/golden/make_impression_eval_golden.py), and the route decision of the overlay's B200ImpressionRunner."""
import math
import os
import types

import numpy as np
import pytest

from tests.impression_oracle import impression_collate, impression_evaluate, impression_history

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "impression_eval.npz")


def _cases(z):
    return sorted({k.split("/")[1] for k in z.files if k.startswith("ev/")})


def test_oracle_equals_reference_evaluate_exactly():
    z = np.load(GOLDEN)
    assert len(_cases(z)) == 5
    for c in _cases(z):
        got = impression_evaluate(z[f"ev/{c}/pred"], z[f"ev/{c}/pos_num"], z[f"ev/{c}/neg_num"], int(z[f"ev/{c}/mp"]),
                                  [int(k) for k in z[f"ev/{c}/topk"]])
        assert list(got) == [str(k) for k in z[f"ev/{c}/keys"]], c
        want = z[f"ev/{c}/values"]
        assert np.array_equal(np.array(list(got.values()), dtype=np.float64), want), c


def _rank_restatement(pred, pos_num, neg_num, mp, topks):
    """include/b200rec.h's per-row contract of b2r_impression_metrics (ranks by counting, no sort), row by row"""
    N, C = pred.shape
    sums = np.zeros(3 * len(topks))
    for r in range(N):
        P, Q = min(int(pos_num[r]), mp), min(int(neg_num[r]), C - mp)
        W = P + Q
        key = [(float(pred[r, c]) if (c < P or mp <= c < mp + Q) else -math.inf) - (1e-6 if c < mp else 0.0)
               for c in range(C)]

        def before(c, j):
            if math.isnan(key[j]):
                return not math.isnan(key[c]) or c < j
            if math.isnan(key[c]):
                return False
            return key[c] > key[j] or (key[c] == key[j] and c < j)

        ranks = sorted(x for x in (sum(before(c, j) for c in range(C)) for j in range(P)) if x < W)
        Pm = len(ranks)
        for i, k in enumerate(topks):
            idcg = sum(1 / math.log2(t + 2) for t in range(min(Pm, k))) or 1.0
            sums[i] += sum(1 / math.log2(x + 2) for x in ranks if x < k) / idcg
            sums[len(topks) + i] += sum((m + 1) / (x + 1) for m, x in enumerate(ranks) if x < k) / min(max(Pm, 1), k)
            sums[2 * len(topks) + i] += float(any(x < k for x in ranks))
    return sums / N


def test_rank_counting_contract_matches_reference():
    z = np.load(GOLDEN)
    for c in _cases(z):
        ks = [int(k) for k in z[f"ev/{c}/topk"]]
        got = _rank_restatement(z[f"ev/{c}/pred"], z[f"ev/{c}/pos_num"], z[f"ev/{c}/neg_num"], int(z[f"ev/{c}/mp"]), ks)
        assert np.abs(got - z[f"ev/{c}/values"]).max() <= 1e-12, c


def test_oracle_refuses_mn_above_mp_as_the_reference_does():
    with pytest.raises(IndexError):
        impression_evaluate(np.zeros((2, 5), np.float32), [1, 1], [3, 3], 2, [1])


def test_host_collate_equals_reference_batches():
    z = np.load(GOLDEN)
    mp, mn, B, H = (int(z[f"col/{k}"]) for k in ("mp", "mn", "B", "history_max"))
    users, position = z["col/user_id"], z["col/position"]
    pp, pf, npt, nf = z["col/pos_ptr"], z["col/pos_flat"], z["col/neg_ptr"], z["col/neg_flat"]
    pos = [pf[pp[i]:pp[i + 1]] for i in range(len(users))]
    neg = [nf[npt[i]:npt[i + 1]] for i in range(len(users))]
    assert max(len(p) for p in pos) > mp and max(len(n) for n in neg) > mn
    hp, hf = z["col/his_ptr"], z["col/his_flat"]
    his = {int(u): [(int(x), 0) for x in hf[hp[i]:hp[i + 1]]] for i, u in enumerate(z["col/his_users"])}
    for tag in ("general", "seq"):
        rows = np.arange(len(users)) if tag == "general" else np.flatnonzero(position > 0)
        assert len(rows) == int(z[f"col/{tag}/rows"])
        for bi, start in enumerate(range(0, len(rows), B)):
            r = rows[start:start + B]
            uid, iid = impression_collate([pos[i] for i in r], [neg[i] for i in r], users[r], mp, mn)
            assert np.array_equal(uid, z[f"col/{tag}/{bi}/user_id"]) and np.array_equal(iid, z[f"col/{tag}/{bi}/item_id"])
            if tag == "seq":
                hi, ln = impression_history(his, users[r], position[r], H)
                assert np.array_equal(hi, z[f"col/{tag}/{bi}/history_items"])
                assert np.array_equal(ln, z[f"col/{tag}/{bi}/lengths"])


# ---- route decision --------------------------------------------------------------------------------------------------

class _StubImpressionRunner:
    """stands in for the reference's ImpressionRunner: records what its evaluate was asked"""

    @staticmethod
    def parse_runner_args(parser):
        return parser

    def __init__(self, args):
        self.eval_batch_size = 4
        self.calls = []

    def evaluate(self, data, topks, metrics, check_sort_idx=0, all=0):
        self.calls.append((check_sort_idx, all))
        return {"host": 1.0}


def _setup(monkeypatch, flag=1, test_all=0, mp=3, mn=3, pos_num=True, rows=2, kernels=True):
    from rechorus_b200 import overlay, runner
    device_calls = []
    monkeypatch.setattr(runner, "evaluate_impression_on_device", lambda r, d, k: device_calls.append(k) or {"dev": 1.0})
    cls = overlay._make_impression_runner_module(_StubImpressionRunner).B200ImpressionRunner
    run = cls(types.SimpleNamespace(device_metrics=flag))
    model = types.SimpleNamespace(test_all=test_all, test_max_pos_item=mp, test_max_neg_item=mn)
    if kernels:
        model.eval_ranks = lambda *a, **k: None
    data = {"user_id": list(range(rows)), "neg_num": [1] * rows}
    if pos_num:
        data["pos_num"] = [1] * rows
    return run, types.SimpleNamespace(model=model, data=data), device_calls


def test_device_route_taken_when_every_condition_holds(monkeypatch):
    run, ds, dev = _setup(monkeypatch, mn=2)
    assert run.evaluate(ds, [5], ["NDCG"]) == {"dev": 1.0} and dev == [[5]] and run.calls == []


@pytest.mark.parametrize("case", ["no_flag", "test_all", "mn_above_mp", "check_sort_idx", "all", "no_pos_num",
                                  "no_rows", "host_model"])
def test_excluded_cases_keep_the_reference_evaluate(monkeypatch, case):
    kw = {"no_flag": dict(flag=0), "test_all": dict(test_all=1), "mn_above_mp": dict(mp=2, mn=3),
          "no_pos_num": dict(pos_num=False), "no_rows": dict(rows=0), "host_model": dict(kernels=False)}.get(case, {})
    run, ds, dev = _setup(monkeypatch, **kw)
    args = {"check_sort_idx": (1, 0), "all": (0, 1)}.get(case, (0, 0))
    assert run.evaluate(ds, [5], ["NDCG"], *args) == {"host": 1.0}
    assert run.calls == [args] and dev == []


def test_parser_knows_device_metrics():
    import argparse

    from rechorus_b200 import overlay
    cls = overlay._make_impression_runner_module(_StubImpressionRunner).B200ImpressionRunner
    a = cls.parse_runner_args(argparse.ArgumentParser()).parse_args(["--device_metrics", "1"])
    assert a.device_metrics == 1
