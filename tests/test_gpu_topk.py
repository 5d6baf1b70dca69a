"""GPU: the top-k recommendation lists (b2r_topk_rows, b2r_mask_clicked, b2r_topk_all_items), the plugin's recommend,
BaseRunner.recommend / save_rec_results against predict + the reference's host sort (main.py:117-132), and the
overlay's --device_rec route through the unchanged main.py."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref", "src")
sys.path.insert(0, HERE)
import topk_oracle as T  # noqa: E402

pytestmark = [pytest.mark.gpu]
DEV = torch.device("cuda", 0)


def _bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


# ---- b2r_topk_rows -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("N,C", [(1, 1), (7, 2), (300, 100), (64, 1024), (5, 5000), (3, 100000), (2, 1000003)])
@pytest.mark.parametrize("k", [1, 10, 100, 1024])
def test_topk_rows_bit_exact(N, C, k):
    from rechorus_b200 import ops
    x = T.planted_rows(np.random.RandomState(N * 7 + C + k), N, C)
    cols, scores = ops.topk_rows(torch.from_numpy(x).to(DEV), k)
    rc, rs = T.topk_rows(x, k)
    assert cols.shape == (N, min(k, C))
    assert np.array_equal(cols.cpu().numpy(), rc)
    assert np.array_equal(_bits(scores.cpu().numpy()), _bits(rs))


def test_topk_rows_sorted_input_worst_case():
    """every element beats the threshold (ascending rows): the buffer flushes every round and stays exact"""
    from rechorus_b200 import ops
    x = np.tile(np.arange(20000, dtype=np.float32), (3, 1))
    cols, _ = ops.topk_rows(torch.from_numpy(x).to(DEV), 1024)
    assert np.array_equal(cols.cpu().numpy(), T.topk_order(x, 1024))


# ---- b2r_mask_clicked --------------------------------------------------------------------------------------------

def _clicked(rng, n_users, n_items, dense_users=()):
    train, residual = {}, {}
    for u in range(n_users):
        if u in dense_users:
            s = set(range(1, n_items)) - set(rng.randint(1, n_items, 3).tolist())
        else:
            s = set(rng.randint(1, n_items, rng.randint(0, 12)).tolist())
        half = len(s) // 2
        lst = sorted(s)
        train[u], residual[u] = set(lst[:half]), set(lst[half:])
    return train, residual


def test_mask_clicked_equals_host_loop():
    from rechorus_b200 import ops
    rng = np.random.RandomState(3)
    n_users, C, N = 40, 500, 70
    train, residual = _clicked(rng, n_users, C, dense_users=(5,))
    users = rng.randint(0, n_users, N)
    users[3] = 5
    pred = rng.standard_normal((N, C)).astype(np.float32)
    ref = pred.copy()
    rows, cols = [], []                                        # BaseRunner.py:244-251
    for i, u in enumerate(users):
        clicked = list(train[u] | residual[u])
        rows.extend([i] * len(clicked))
        cols.extend(clicked)
    ref[rows, cols] = -np.inf
    got = torch.from_numpy(pred).to(DEV)
    ops.mask_clicked(got, torch.from_numpy(users).to(DEV), ops.ClickedSets(train, residual, n_users, DEV))
    assert np.array_equal(_bits(got.cpu().numpy()), _bits(ref))
    ops.check_ids(DEV)


# ---- b2r_topk_all_items ------------------------------------------------------------------------------------------

def _all_items_case(rng, B, n_items, d, integer, dense_users=()):
    n_users = B + 3
    if integer:
        q = rng.randint(-3, 4, (B, d)).astype(np.float32)
        table = rng.randint(-3, 4, (n_items, d)).astype(np.float32)
    else:
        q = rng.standard_normal((B, d)).astype(np.float32)
        table = rng.standard_normal((n_items, d)).astype(np.float32)
    users = rng.permutation(n_users)[:B].astype(np.int64)
    train, residual = _clicked(rng, n_users, n_items, dense_users=[users[i] for i in dense_users])
    target = rng.randint(1, n_items, B).astype(np.int64) if n_items > 1 else np.zeros(B, np.int64)
    for b in range(B):                                          # the target is one of the residual clicks
        if n_items > 1:
            residual[users[b]].add(int(target[b]))
    clicked = [sorted(train[u] | residual[u]) for u in users]
    return q, table, users, target, train, residual, clicked


def _run_all_items(q, table, users, target, train, residual, k):
    from rechorus_b200 import ops
    cs = ops.ClickedSets(train, residual, int(max(users.max() + 1, len(train))), DEV)
    items, scores = ops.topk_all_items(torch.from_numpy(q).to(DEV), torch.from_numpy(table).to(DEV),
                                       torch.from_numpy(target).to(DEV), torch.from_numpy(users).to(DEV), cs, k)
    ops.check_ids(DEV)
    return items.cpu().numpy(), scores.cpu().numpy()


@pytest.mark.parametrize("n_items,d,k", [(2, 4, 1), (2, 20, 100), (130, 4, 100), (130, 64, 1024), (4097, 20, 1),
                                         (4097, 128, 100), (4097, 64, 1024), (100003, 64, 100), (100003, 4, 1024)])
def test_topk_all_items_integer_scores_bit_exact(n_items, d, k):
    """integer-valued q and table: every score exact in fp32, ties common; some users clicked nearly everything"""
    rng = np.random.RandomState(n_items + d + k)
    B = 133                                                     # not a multiple of the 128-row tile
    q, table, users, target, train, residual, clicked = _all_items_case(rng, B, n_items, d, True, dense_users=(0, 77))
    items, scores = _run_all_items(q, table, users, target, train, residual, k)
    S = (q.astype(np.float64) @ table.astype(np.float64).T).astype(np.float32)
    m = T.test_all_matrix(S, target, clicked)
    cols, ref_scores = T.topk_rows(m, k)
    ref_items = np.where(cols == 0, target[:, None], cols)
    assert items.shape == (B, min(k, n_items))
    assert np.array_equal(items, ref_items)
    assert np.array_equal(_bits(scores), _bits(ref_scores))


def test_topk_all_items_random_floats_agree_with_rank_and_matmul():
    from rechorus_b200 import ops
    rng = np.random.RandomState(11)
    B, n_items, d, k = 300, 20011, 64, 100
    q, table, users, target, train, residual, clicked = _all_items_case(rng, B, n_items, d, False)
    items, scores = _run_all_items(q, table, users, target, train, residual, k)
    items2, scores2 = _run_all_items(q, table, users, target, train, residual, k)
    assert np.array_equal(items, items2) and np.array_equal(_bits(scores), _bits(scores2))      # two runs bit-identical
    # the target's position equals rank_all_items' rank wherever rank <= k
    mr = np.concatenate([[b] * len(c) for b, c in enumerate(clicked)]).astype(np.int64)
    mi = np.concatenate([c for c in clicked]).astype(np.int64)
    rank = ops.rank_all_items(torch.from_numpy(q).to(DEV), torch.from_numpy(table).to(DEV),
                              torch.from_numpy(target).to(DEV), torch.from_numpy(mr).to(DEV),
                              torch.from_numpy(mi).to(DEV)).cpu().numpy()
    for b in range(B):
        pos = np.flatnonzero(items[b] == target[b])
        if rank[b] <= k:
            assert len(pos) >= 1 and pos[0] + 1 == rank[b], (b, rank[b], pos)
        else:
            assert target[b] not in items[b]
    # lists vs a torch fp32 matmul + stable sort: only swaps of entries closer than 1e-5 of the row's max |score|
    S = (torch.from_numpy(q) @ torch.from_numpy(table).T).numpy()
    m = T.test_all_matrix(S, target, clicked)
    order = T.topk_order(m, n_items)
    ref_sorted = np.take_along_axis(m, order, axis=1)
    for b in range(B):
        tol = 1e-5 * np.abs(S[b]).max()
        ref_items = np.where(order[b] == 0, target[b], order[b])
        assert np.abs(scores[b] - ref_sorted[b, :k]).max() <= 1e-5 * max(1.0, np.abs(S[b]).max())
        pos_in_ref = {int(c): p for p, c in enumerate(order[b])}
        for t in np.flatnonzero(items[b] != ref_items[:k]):
            col = 0 if items[b, t] == target[b] else int(items[b, t])   # the target's own column is masked
            p = pos_in_ref[col]
            assert abs(ref_sorted[b, p] - ref_sorted[b, t]) <= tol, (b, t)


# ---- plugin.recommend / BaseRunner.recommend / save_rec_results -------------------------------------------------

def _corpus():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import fit_corpus
    return fit_corpus.build()


MODELS = {
    "BPRMF": ["--emb_size", "64"],
    "NeuMF": ["--emb_size", "32", "--layers", "[32, 16]"],
    "SASRec": ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "8"],
}


def _setup(name, test_all):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    p = cls.parse_model_args(p)
    a = p.parse_args([*MODELS[name], "--num_workers", "0", "--eval_batch_size", "32", "--test_all", str(test_all)])
    a.device, a.model_path, a.log_file = DEV, "/tmp/_b2r_topk.pt", ""
    corpus = _corpus()
    torch.manual_seed(0)
    model = cls(a, corpus).to(DEV)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(30.0)                                       # trained-scale scores, few near-ties
    ds = cls.Dataset(model, corpus, "test")
    ds.prepare()
    return model, ds, BaseRunner(a)


def _host_lists(runner, ds, k):
    """main.py:121-126: predict, then the Python sort of zip(item_id, prediction) row by row"""
    preds = runner.predict(ds)
    items, scores = [], []
    for i in range(len(ds)):
        info = ds[i]
        lst = sorted(zip(info["item_id"], preds[i]), key=lambda x: x[1], reverse=True)[:k]
        items.append([x[0] for x in lst])
        scores.append([x[1] for x in lst])
    return np.array(items, dtype=np.int64), np.array(scores, dtype=np.float32)


def _close_lists(items, scores, ref_items, ref_scores):
    tol = 1e-5 * max(1.0, float(np.abs(ref_scores[np.isfinite(ref_scores)]).max()))
    fin = np.isfinite(ref_scores)
    assert (np.isfinite(scores) == fin).all()
    assert not fin.any() or np.abs(scores[fin] - ref_scores[fin]).max() <= tol
    for b, t in zip(*np.nonzero(items != ref_items)):
        hits = np.flatnonzero(ref_items[b] == items[b, t])
        assert len(hits) and abs(ref_scores[b, hits[0]] - ref_scores[b, t]) <= tol, (b, t)


@pytest.mark.parametrize("name", ["BPRMF", "NeuMF", "SASRec"])
@pytest.mark.parametrize("test_all", [0, 1])
def test_runner_recommend_equals_predict_and_host_sort(name, test_all):
    model, ds, runner = _setup(name, test_all)
    k = 20
    users, items, scores = runner.recommend(ds, k)
    ref_items, ref_scores = _host_lists(runner, ds, k)
    assert users == list(ds.data["user_id"])
    assert items.dtype == np.int64 and scores.dtype == np.float32 and items.shape == ref_items.shape
    exact = name == "NeuMF" or (name == "BPRMF" and not test_all)
    if exact:
        assert np.array_equal(items, ref_items)
        assert np.array_equal(_bits(scores), _bits(ref_scores))
    else:
        _close_lists(items, scores, ref_items, ref_scores)


def test_save_rec_results_writes_the_reference_csv(tmp_path):
    """the TopK branch of main.py:117-132, written from predict + the host sort vs from recommend: same bytes"""
    model, ds, runner = _setup("NeuMF", 0)
    ref_items, ref_scores = _host_lists(runner, ds, 100)
    rec_df = pd.DataFrame(columns=["user_id", "rec_items", "rec_predictions"])
    rec_df["user_id"] = [ds[i]["user_id"] for i in range(len(ds))]
    rec_df["rec_items"] = [list(r) for r in ref_items]
    rec_df["rec_predictions"] = [list(r) for r in ref_scores]
    ref_path, path = str(tmp_path / "ref.csv"), str(tmp_path / "out" / "rec.csv")
    rec_df.to_csv(ref_path, sep="\t", index=False)
    runner.save_rec_results(ds, path, 100, sep="\t")
    assert open(path, "rb").read() == open(ref_path, "rb").read()


# ---- overlay: --device_rec 1 through the unchanged main.py -------------------------------------------------------

N_USERS, N_ITEMS, ROWS, N_EVAL, N_NEG = 60, 90, 1500, 120, 29


def _dataset(root):
    rng = np.random.RandomState(7)                              # tests/test_gpu_overlay.py's tiny dataset
    d = os.path.join(root, "data", "tiny")
    os.makedirs(d)
    df = pd.DataFrame({"user_id": rng.randint(1, N_USERS, ROWS), "item_id": rng.randint(1, N_ITEMS, ROWS),
                       "time": np.arange(ROWS)})
    tr = df.iloc[:ROWS - 2 * N_EVAL]
    tr.to_csv(os.path.join(d, "train.csv"), sep="\t", index=False)
    seen = set(tr.user_id)
    for name, part in (("dev", df.iloc[ROWS - 2 * N_EVAL:ROWS - N_EVAL]), ("test", df.iloc[ROWS - N_EVAL:])):
        part = part[part.user_id.isin(seen)].copy()
        part["neg_items"] = [str(list(rng.randint(1, N_ITEMS, N_NEG))) for _ in range(len(part))]
        part.to_csv(os.path.join(d, name + ".csv"), sep="\t", index=False)


def _main(tmp, tag, model, flags, mp, train):
    cwd = os.path.join(tmp, tag, "src")
    os.makedirs(cwd)
    lf = os.path.join(tmp, tag, "log", "run.txt")
    cmd = [sys.executable, "-m", "rechorus_b200.overlay", "--ref", REF, "--model_name", model, "--dataset", "tiny",
           "--path", os.path.join(tmp, "data") + "/", "--gpu", "0", "--num_workers", "0", "--epoch", "1",
           "--early_stop", "0", "--batch_size", "128", "--eval_batch_size", "64", "--lr", "0.01", "--l2", "0",
           "--topk", "5,10", "--model_path", mp, "--log_file", lf, "--regenerate", "1", "--random_seed", "0",
           "--load", str(1 - train), "--train", str(train), "--save_final_results", str(1 - train), *flags]
    res = subprocess.run(cmd, cwd=cwd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True,
                         timeout=900)
    assert res.returncode == 0, (res.stdout + res.stderr)[-3000:]
    out_dir = os.path.join(tmp, tag, "log", "run")
    return {ph: os.path.join(out_dir, f"rec-{model}-{ph}.csv") for ph in ("dev", "test")}


OVERLAY_CASES = [("BPRMF", ["--emb_size", "64"], 0, True), ("NeuMF", ["--emb_size", "32", "--layers", "[32, 16]"], 0, True),
                 ("NeuMF", ["--emb_size", "32", "--layers", "[32, 16]"], 1, True), ("BPRMF", ["--emb_size", "64"], 1, False),
                 ("SASRec", ["--emb_size", "32", "--num_heads", "2", "--history_max", "8"], 0, False)]


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "main.py")),
                    reason="no unmodified reference staged in oracle/_ref (build() without the checkout)")
@pytest.mark.parametrize("model,flags,test_all,exact", OVERLAY_CASES)
def test_overlay_device_rec_csv_matches_reference_route(tmp_path, model, flags, test_all, exact):
    tmp = str(tmp_path)
    _dataset(tmp)
    flags = [*flags, "--test_all", str(test_all)]
    mp = os.path.join(tmp, "model.pt")
    _main(tmp, "train", model, flags, mp, 1)
    host = _main(tmp, "host", model, flags, mp, 0)
    dev = _main(tmp, "dev", model, flags + ["--device_rec", "1"], mp, 0)
    for ph in ("dev", "test"):
        a, b = open(host[ph], "rb").read(), open(dev[ph], "rb").read()
        if exact:
            assert a == b, ph
            continue
        ha, hb = pd.read_csv(host[ph], sep="\t"), pd.read_csv(dev[ph], sep="\t")
        assert list(ha.columns) == list(hb.columns) and (ha.user_id.values == hb.user_id.values).all()
        parse_i = lambda s: np.array([int(t) for t in s.replace("np.int64(", "").replace(")", "").strip("[]").split(",")])
        parse_f = lambda s: np.array([float(t) for t in s.replace("np.float32(", "").replace(")", "").strip("[]").split(",")])
        items = np.stack([parse_i(s) for s in hb.rec_items])
        ref_items = np.stack([parse_i(s) for s in ha.rec_items])
        scores = np.stack([parse_f(s) for s in hb.rec_predictions]).astype(np.float32)
        ref_scores = np.stack([parse_f(s) for s in ha.rec_predictions]).astype(np.float32)
        _close_lists(items, scores, ref_items, ref_scores)
