"""GPU: impression evaluation on the device -- b2r_impression_metrics against the reference's evaluate (fixture) and the
NumPy oracle on seeded shapes, determinism, b2r_collate_impression / the history collate against the reference's batches,
and runner.evaluate_impression_on_device for BPRMFImpression and SASRecImpression against the host route."""
import argparse
import types

import numpy as np
import pytest
import torch

from tests.impression_oracle import impression_collate, impression_evaluate, impression_history
from tests.test_impression_eval_cpu import GOLDEN, _cases

pytestmark = [pytest.mark.gpu]
DEV = torch.device("cuda", 0)


def _device_metrics(pred, pos_num, neg_num, mp, ks, B=None):
    """{key: value} from ops.impression_metrics over batches of B rows (one batch when B is None)"""
    from rechorus_b200 import ops
    pred_d = torch.from_numpy(np.ascontiguousarray(pred)).to(DEV)
    pn, nn = torch.from_numpy(np.asarray(pos_num, np.int64)).to(DEV), torch.from_numpy(np.asarray(neg_num, np.int64)).to(DEV)
    N = pred.shape[0]
    B = B or N
    acc = torch.zeros(3 * len(ks), dtype=torch.float64, device=DEV)
    for s in range(0, N, B):
        ops.impression_metrics(pred_d[s:s + B], pn[s:s + B], nn[s:s + B], mp, ks, acc)
    sums = acc.cpu().numpy()
    out = {}
    for m, name in enumerate(("NDCG", "MAP", "HR")):
        for i, k in enumerate(ks):
            out[f"{name}@{k}"] = sums[m * len(ks) + i] / N
    return out, sums


def _close(got, want, tol=1e-12):
    assert list(got) == list(want)
    diff = max(abs(got[k] - want[k]) for k in want)
    assert diff <= tol, (diff, got, want)


def test_kernel_matches_reference_fixture():
    z = np.load(GOLDEN)
    for c in _cases(z):
        ks = [int(k) for k in z[f"ev/{c}/topk"]]
        want = dict(zip([str(k) for k in z[f"ev/{c}/keys"]], z[f"ev/{c}/values"]))
        for B in (None, 64, 7):
            got, _ = _device_metrics(z[f"ev/{c}/pred"], z[f"ev/{c}/pos_num"], z[f"ev/{c}/neg_num"], int(z[f"ev/{c}/mp"]),
                                     ks, B)
            _close(got, want)


def _random_case(seed, N, mp, mn, special):
    rng = np.random.RandomState(seed)
    C = mp + mn
    pred = rng.randint(-3, 4, (N, C)).astype(np.float32) if seed % 2 else rng.randn(N, C).astype(np.float32)
    if special:
        pick = rng.rand(N, C)
        pred[pick < 0.05] = -np.inf
        pred[(pick >= 0.05) & (pick < 0.08)] = np.nan
    pos_num = rng.randint(0, mp + 3, N)
    neg_num = rng.randint(0, mn + 3, N)
    return pred, pos_num, neg_num


# (mp, mn): C from 2 to 600; mn > mp is outside the reference (it raises there) but inside the kernel's contract, which
# the oracle computes all the same with allow_wide_neg
SHAPES = [(1, 1), (1, 40), (3, 0), (3, 3), (3, 125), (20, 20), (20, 7), (20, 300), (1, 599), (20, 580)]


@pytest.mark.parametrize("mp,mn", SHAPES)
def test_kernel_matches_oracle_on_seeded_shapes(mp, mn):
    for seed, special in ((mp * 1000 + mn, False), (mp * 1000 + mn + 1, True)):
        pred, pn, nn = _random_case(seed, 333, mp, mn, special)
        ks = [1, 2, 5, 10, 50, 1000]
        want = impression_evaluate(pred, pn, nn, mp, ks, allow_wide_neg=True)
        got, _ = _device_metrics(pred, pn, nn, mp, ks, B=128)
        _close(got, want)


def test_one_large_batch_and_identical_bits():
    pred, pn, nn = _random_case(77, 200_000, 20, 20, True)
    ks = [1, 5, 10, 20]
    want = impression_evaluate(pred, pn, nn, 20, ks)
    got, s1 = _device_metrics(pred, pn, nn, 20, ks)
    _close(got, want)
    _, s2 = _device_metrics(pred, pn, nn, 20, ks)
    assert s1.tobytes() == s2.tobytes()


def test_bad_arguments_are_rejected():
    from rechorus_b200 import lib, ops
    L = lib.load()
    z = torch.zeros((2, 4), device=DEV)
    n = torch.ones(2, dtype=torch.int64, device=DEV)
    acc = torch.zeros(3, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError):
        ops.impression_metrics(z, n, n, 5, [1], acc)                   # mp > C
    with pytest.raises(ValueError):
        ops.impression_metrics(z, n, n, 2, [0], acc)                   # k < 1
    import ctypes as C
    ks = (C.c_int * 1)(0)
    assert L.b2r_impression_metrics(z.data_ptr(), 4, 2, 4, 2, n.data_ptr(), n.data_ptr(), ks, 1, acc.data_ptr(),
                                    acc.data_ptr(), 1 << 20, None) == -1
    ks = (C.c_int * 1)(1)
    assert L.b2r_impression_metrics(z.data_ptr(), 4, 2, 4, 5, n.data_ptr(), n.data_ptr(), ks, 1, acc.data_ptr(),
                                    acc.data_ptr(), 1 << 20, None) == -1
    assert L.b2r_impression_metrics(z.data_ptr(), 4, 2, 0, 0, n.data_ptr(), n.data_ptr(), ks, 1, acc.data_ptr(),
                                    acc.data_ptr(), 1 << 20, None) == -1
    assert L.b2r_impression_metrics(None, 4, 2, 4, 2, n.data_ptr(), n.data_ptr(), ks, 1, acc.data_ptr(),
                                    acc.data_ptr(), 1 << 20, None) == -1
    assert L.b2r_collate_impression(None, None, None, None, None, 3, 0, 1, 1, 1, None, None, None, None) == -1


# ---- device batches against the reference's collate ------------------------------------------------------------------

def _fixture_dataset(z, tag, mp=None, mn=None):
    users, position = z["col/user_id"], z["col/position"]
    pp, pf, npt, nf = z["col/pos_ptr"], z["col/pos_flat"], z["col/neg_ptr"], z["col/neg_flat"]
    rows = np.arange(len(users)) if tag == "general" else np.flatnonzero(position > 0)
    hp, hf = z["col/his_ptr"], z["col/his_flat"]
    his = {int(u): {"pos": [(int(x), 0) for x in hf[hp[i]:hp[i + 1]]], "neg": []} for i, u in enumerate(z["col/his_users"])}
    data = {"user_id": [int(users[r]) for r in rows], "pos_items": [list(pf[pp[r]:pp[r + 1]]) for r in rows],
            "neg_items": [list(nf[npt[r]:npt[r + 1]]) for r in rows], "position": [int(position[r]) for r in rows]}
    data["pos_num"] = [len(x) for x in data["pos_items"]]
    data["neg_num"] = [len(x) for x in data["neg_items"]]
    model = types.SimpleNamespace(device=DEV, test_all=0, test_max_pos_item=mp or int(z["col/mp"]),
                                  test_max_neg_item=mn or int(z["col/mn"]))
    if tag == "seq":
        model.history_max = int(z["col/history_max"])
    corpus = types.SimpleNamespace(user_his=his, n_users=int(z["col/n_users"]))
    return types.SimpleNamespace(model=model, corpus=corpus, data=data, phase="dev")


@pytest.mark.parametrize("tag", ["general", "seq"])
def test_device_batches_equal_reference_collate(tag):
    from rechorus_b200.runner import device_impression_batches
    z = np.load(GOLDEN)
    ds = _fixture_dataset(z, tag)
    n = 0
    for bi, (start, feed) in enumerate(device_impression_batches(ds, int(z["col/B"]))):
        assert start == bi * int(z["col/B"])
        assert np.array_equal(feed["user_id"].cpu().numpy(), z[f"col/{tag}/{bi}/user_id"])
        assert np.array_equal(feed["item_id"].cpu().numpy(), z[f"col/{tag}/{bi}/item_id"])
        if tag == "seq":
            assert np.array_equal(feed["history_items"].cpu().numpy(), z[f"col/{tag}/{bi}/history_items"])
            assert np.array_equal(feed["lengths"].cpu().numpy(), z[f"col/{tag}/{bi}/lengths"])
        n += 1
    assert n == (int(z[f"col/{tag}/rows"]) + int(z["col/B"]) - 1) // int(z["col/B"])


# ---- evaluate_impression_on_device against the host route ------------------------------------------------------------

N_USERS, N_ITEMS = 50, 120
MODELS = {"BPRMFImpression": ["--emb_size", "64"],
          "SASRecImpression": ["--emb_size", "64", "--num_layers", "1", "--num_heads", "1", "--history_max", "20"]}


def _impression_dataset(name, N, mp, mn, seed, bad_user=False):
    rng = np.random.RandomState(seed)
    his = {u: {"pos": [(int(i), t) for t, i in enumerate(rng.randint(1, N_ITEMS, rng.randint(1, 40)))], "neg": []}
           for u in range(1, N_USERS)}
    users = rng.randint(1, N_USERS, N)
    if bad_user:
        users[N // 2] = N_USERS + 3
        his[N_USERS + 3] = {"pos": [(1, 0)], "neg": []}
    data = {"user_id": [int(u) for u in users],
            "pos_items": [list(rng.randint(1, N_ITEMS, rng.randint(1, mp + 5))) for _ in range(N)],
            "neg_items": [list(rng.randint(1, N_ITEMS, rng.randint(1, mn + 5))) for _ in range(N)],
            "position": [int(rng.randint(1, len(his[int(u)]["pos"]) + 1)) for u in users]}
    data["pos_num"] = [len(x) for x in data["pos_items"]]
    data["neg_num"] = [len(x) for x in data["neg_items"]]
    return data, his


def _model(name, mp, mn):
    from rechorus_b200 import plugin
    cls = getattr(plugin, name)
    a = cls.parse_model_args(argparse.ArgumentParser()).parse_args(
        [*MODELS[name], "--test_max_pos_item", str(mp), "--test_max_neg_item", str(mn)])
    a.device, a.model_path = DEV, "/tmp/_b2r_imp_eval.pt"
    torch.manual_seed(3)
    m = cls(a, types.SimpleNamespace(n_users=N_USERS, n_items=N_ITEMS)).to(DEV)
    with torch.no_grad():
        for q in m.parameters():
            q.mul_(30.0)                                                  # spread the scores
    return m


def _host_predictions(model, ds, B):
    """the host route's predictions: the oracle's collate per batch, then the model's forward"""
    d, preds = ds.data, []
    mp, mn = model.test_max_pos_item, model.test_max_neg_item
    for s in range(0, len(d["user_id"]), B):
        r = range(s, min(len(d["user_id"]), s + B))
        uid, iid = impression_collate([d["pos_items"][i] for i in r], [d["neg_items"][i] for i in r],
                                      [d["user_id"][i] for i in r], mp, mn)
        feed = {"user_id": torch.from_numpy(uid).to(DEV), "item_id": torch.from_numpy(iid).to(DEV),
                "batch_size": len(r), "phase": "dev"}
        if hasattr(model, "history_max"):
            his = {u: h["pos"] for u, h in ds.corpus.user_his.items()}
            hi, ln = impression_history(his, uid, [d["position"][i] for i in r], model.history_max)
            feed["history_items"], feed["lengths"] = torch.from_numpy(hi).to(DEV), torch.from_numpy(ln).to(DEV)
        preds.append(model.inference(feed)["prediction"].cpu().numpy())
    return np.concatenate(preds)


@pytest.mark.parametrize("name", list(MODELS))
def test_evaluate_on_device_equals_host_route(name):
    from torch.utils.data import DataLoader

    from rechorus_b200.runner import evaluate_impression_on_device
    mp, mn, N, B = 6, 4, 517, 64
    data, his = _impression_dataset(name, N, mp, mn, seed=len(name))
    model = _model(name, mp, mn)
    ds = types.SimpleNamespace(model=model, data=data, phase="dev",
                               corpus=types.SimpleNamespace(user_his=his, n_users=N_USERS, n_items=N_ITEMS))
    ks = [1, 3, 5, 10]
    runner = types.SimpleNamespace(eval_batch_size=B)
    torch.manual_seed(11)
    got = evaluate_impression_on_device(runner, ds, ks)
    after_device = torch.get_rng_state()
    want = impression_evaluate(_host_predictions(model, ds, B), data["pos_num"], data["neg_num"], mp, ks)
    _close(got, want)
    assert all(isinstance(v, np.float64) for v in got.values())
    # the host route's DataLoader iterator draws one seed from the global CPU generator
    torch.manual_seed(11)
    iter(DataLoader(list(range(N)), batch_size=B, shuffle=False, num_workers=0))
    assert torch.equal(after_device, torch.get_rng_state())
    # a second evaluation reuses the cached phase state and gives the same bits
    again = evaluate_impression_on_device(runner, ds, ks)
    assert [v.tobytes() for v in again.values()] == [v.tobytes() for v in got.values()]


def test_out_of_range_user_raises_at_the_poll():
    from rechorus_b200 import ops
    from rechorus_b200.runner import evaluate_impression_on_device
    data, his = _impression_dataset("BPRMFImpression", 40, 3, 3, seed=5, bad_user=True)
    model = _model("BPRMFImpression", 3, 3)
    ds = types.SimpleNamespace(model=model, data=data, phase="dev",
                               corpus=types.SimpleNamespace(user_his=his, n_users=N_USERS, n_items=N_ITEMS))
    ops.poll_ids(DEV)
    with pytest.raises(IndexError):
        evaluate_impression_on_device(types.SimpleNamespace(eval_batch_size=16), ds, [1, 5])
