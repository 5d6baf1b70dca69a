"""GPU: evaluation on device-built batches -- b2r_rank_all_items_clicked (the test_all ranks masked from the clicked-item
CSR) against the COO route, every device-built evaluation batch against collate_batch, --device_metrics 1 against the host
predict + evaluate_method route, a device evaluation with the host batch path disabled, a large catalogue, and the overlay's
main.py with and without --device_metrics 1."""
import argparse
import os
import re
import subprocess
import sys
import types

import numpy as np
import pandas as pd
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref", "src")
sys.path.insert(0, os.path.join(HERE, "golden"))
from rechorus_b200.runner import device_eval_batches  # noqa: E402

pytestmark = [pytest.mark.gpu]
DEV = torch.device("cuda", 0)


# ---- b2r_rank_all_items_clicked ----------------------------------------------------------------------------------

def _kernel_case(rng, B, n_items, d, integer):
    n_users = B + 5
    if integer:                                                 # exact scores: ties with s0 are common
        q = rng.randint(-2, 3, (B, d)).astype(np.float32)
        table = rng.randint(-2, 3, (n_items, d)).astype(np.float32)
    else:
        q = rng.standard_normal((B, d)).astype(np.float32)
        table = rng.standard_normal((n_items, d)).astype(np.float32)
    users = rng.randint(0, n_users, B).astype(np.int64)
    target = rng.randint(1, max(n_items, 2), B).astype(np.int64) % n_items
    train, residual = {}, {}
    for u in range(n_users):
        if u % 4 == 0:
            continue                                            # users without clicks
        s = set(rng.randint(1, max(n_items, 2), rng.randint(0, 40)).tolist())
        s |= {0, n_items, n_items + 7} if u % 3 == 0 else set()  # ids outside the candidate columns
        lst = sorted(s)
        train[u], residual[u] = set(lst[::2]), set(lst[1::2])
    for b in range(0, B, 2):                                    # the target inside its own clicked set
        residual.setdefault(int(users[b]), set()).add(int(target[b]))
    return q, table, users, target, train, residual, n_users


def _coo(users, train, residual):
    rows, cols = [], []
    for b, u in enumerate(users):
        c = sorted(train.get(int(u), set()) | residual.get(int(u), set()))
        rows.extend([b] * len(c))
        cols.extend(c)
    return np.array(rows, dtype=np.int64), np.array(cols, dtype=np.int64)


@pytest.mark.parametrize("B,n_items", [(1, 2), (37, 130), (133, 1000), (300, 4097)])
@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("integer", [True, False])
def test_rank_all_items_clicked_equals_coo_route(B, n_items, d, integer):
    from rechorus_b200 import ops
    rng = np.random.RandomState(B * 31 + n_items + d + integer)
    q, table, users, target, train, residual, n_users = _kernel_case(rng, B, n_items, d, integer)
    rows, cols = _coo(users, train, residual)
    t = lambda a: torch.from_numpy(a).to(DEV)
    cs = ops.ClickedSets(train, residual, n_users, DEV)
    got = ops.rank_all_items_clicked(t(q), t(table), t(target), t(users), cs).cpu().numpy()
    ref = ops.rank_all_items(t(q), t(table), t(target), t(rows) if len(rows) else None,
                             t(cols) if len(cols) else None).cpu().numpy()
    ops.check_ids(DEV)
    assert np.array_equal(got, ref)
    if integer:                                                 # and the host definition, exactly
        S = q.astype(np.float64) @ table.astype(np.float64).T
        m = S.copy()
        m[:, 0] = -np.inf
        keep = (cols >= 1) & (cols < n_items)
        m[rows[keep], cols[keep]] = -np.inf
        want = 1 + (m >= S[np.arange(B), target][:, None]).sum(1)
        assert np.array_equal(got, want)


def test_rank_all_items_clicked_flags_out_of_range_user():
    from rechorus_b200 import ops
    rng = np.random.RandomState(5)
    q, table, users, target, train, residual, n_users = _kernel_case(rng, 40, 300, 64, False)
    users[7] = n_users + 3
    users[9] = -1
    t = lambda a: torch.from_numpy(a).to(DEV)
    ops.rank_all_items_clicked(t(q), t(table), t(target), t(users), ops.ClickedSets(train, residual, n_users, DEV))
    with pytest.raises(IndexError):
        ops.check_ids(DEV)
    ops.check_ids(DEV)                                          # the raise reset the counter


# ---- the stand-alone runner on fit_corpus -----------------------------------------------------------------------

MODELS = {
    "BPRMF": ["--emb_size", "64"],
    "NeuMF": ["--emb_size", "32", "--layers", "[32, 16]"],
    "SASRec": ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "8"],
    "SASRec_whole": ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "0"],
}


def _setup(name, test_all, eval_bs=7, scale=20.0):
    import fit_corpus
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name.split("_")[0])
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    p = cls.parse_model_args(p)
    a = p.parse_args([*MODELS[name], "--num_workers", "0", "--eval_batch_size", str(eval_bs), "--test_all",
                      str(test_all), "--topk", "1,5,10"])
    a.device, a.model_path, a.log_file = DEV, "/tmp/_b2r_deval.pt", ""
    corpus = fit_corpus.build()
    for u in range(0, corpus.n_users, 3):                       # residual clicks beyond the eval rows' own items
        corpus.residual_clicked_set[u] = corpus.residual_clicked_set[u] | {1 + (u * 7) % (corpus.n_items - 1), 2}
    torch.manual_seed(0)
    model = cls(a, corpus).to(DEV)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(scale)                                     # spread the scores: rank gaps far above fp32 rounding
    ds = cls.Dataset(model, corpus, "dev")
    ds.prepare()
    model.eval()
    return model, ds, BaseRunner(a)


CASES = [(m, t) for m in MODELS for t in (0, 1)]
# SASRec's position table has history_max + 1 rows (SASRec.py:43), so its forward needs history_max > 0; the batches of
# history_max <= 0 (the whole history) are checked above all the same
MODEL_CASES = [(m, t) for m, t in CASES if m != "SASRec_whole"]


@pytest.mark.parametrize("name,test_all", CASES)
def test_device_batches_equal_collate_batch(name, test_all):
    model, ds, runner = _setup(name, test_all)
    N, B = len(ds), runner.eval_batch_size
    assert N % B != 0
    n = 0
    for bi, (feed, clicked) in enumerate(device_eval_batches(ds, runner.eval_batch_size)):
        rows = list(range(bi * B, min(N, bi * B + B)))
        ref = ds.collate_batch([ds[i] for i in rows])
        assert feed["batch_size"] == ref["batch_size"] == len(rows) and feed["phase"] == ref["phase"]
        assert (clicked is not None) == bool(test_all)
        keys = ["user_id", "item_id"] + (["history_items", "lengths"] if "history_items" in ref else [])
        for k in keys:
            got = feed[k].cpu()
            if k == "item_id" and test_all and model.has_query_rows():
                assert torch.equal(got, ref[k][:, :1]), (bi, k)  # a dot-product model needs the targets only
                continue
            assert got.dtype == ref[k].dtype and got.shape == ref[k].shape, (bi, k, got.shape, ref[k].shape)
            assert torch.equal(got, ref[k]), (bi, k)
        n += len(rows)
    assert n == N


def _device_ranks(runner, ds):
    return np.concatenate([ds.model.eval_ranks(f, clicked=c).cpu().numpy()
                           for f, c in device_eval_batches(ds, runner.eval_batch_size)])


@pytest.mark.parametrize("name,test_all", MODEL_CASES)
def test_device_metrics_equal_host_route(name, test_all):
    model, ds, runner = _setup(name, test_all)
    preds = runner.predict(ds)
    host = runner.evaluate_method(preds, [1, 5, 10], ["HR", "NDCG"])
    runner.device_metrics = 1
    dev = runner.evaluate(ds, [1, 5, 10], ["HR", "NDCG"])
    assert set(host) == set(dev)
    for k in host:
        assert abs(host[k] - dev[k]) <= 1e-12, (k, host[k], dev[k])
    want = (preds >= preds[:, 0].reshape(-1, 1)).sum(axis=-1)
    assert np.array_equal(_device_ranks(runner, ds), want)
    if name == "SASRec":                                       # history_max 8: the Linear layers' SGEMM class
        assert max(int(f["history_items"].shape[1]) for f, _ in device_eval_batches(ds, runner.eval_batch_size)) < 16


@pytest.mark.parametrize("name,test_all", [("BPRMF", 1), ("NeuMF", 1), ("SASRec", 0), ("SASRec", 1)])
def test_device_evaluation_builds_no_host_batches(name, test_all, monkeypatch):
    from rechorus_b200 import plugin, runner as R
    model, ds, runner = _setup(name, test_all)
    host = runner.evaluate(ds, [5, 10], ["HR", "NDCG"])

    def refuse(*a, **k):
        raise AssertionError("host batch path used")

    monkeypatch.setattr(plugin.BaseModel.Dataset, "__getitem__", refuse)
    monkeypatch.setattr(plugin.BaseModel.Dataset, "collate_batch", refuse)
    monkeypatch.setattr(R, "DataLoader", refuse)
    runner.device_metrics = 1
    dev = runner.evaluate(ds, [5, 10], ["HR", "NDCG"])
    for k in host:
        assert abs(host[k] - dev[k]) <= 1e-12, k
    runner.recommend(ds, 10)


def test_large_catalogue_test_all_ranks_equal_matmul_reference():
    """BPRMF under test_all at 300k items: integer-valued tables make every score exact, so the ranks must equal a
    float64 matmul + mask + count reference, ties included"""
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    rng = np.random.RandomState(9)
    n_users, n_items, rows = 500, 300_000, 333
    ev = pd.DataFrame({"user_id": rng.randint(1, n_users, rows), "item_id": rng.randint(1, n_items, rows)})
    ev["neg_items"] = [[1] for _ in range(rows)]
    train = {u: set(rng.randint(1, n_items, rng.randint(0, 300)).tolist()) for u in range(n_users)}
    train[int(ev.user_id[0])] |= set(range(1, 60_000))         # one user clicked a fifth of the catalogue
    residual = {u: set() for u in range(n_users)}
    for u, i in zip(ev.user_id, ev.item_id):
        residual[int(u)].add(int(i))
    corpus = types.SimpleNamespace(n_users=n_users, n_items=n_items, data_df={"dev": ev}, train_clicked_set=train,
                                   residual_clicked_set=residual)
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    p = plugin.BPRMF.parse_model_args(p)
    a = p.parse_args(["--emb_size", "64", "--test_all", "1", "--eval_batch_size", "128", "--device_metrics", "1",
                      "--topk", "1,10,100"])
    a.device, a.model_path, a.log_file = DEV, "/tmp/_b2r_deval_big.pt", ""
    model = plugin.BPRMF(a, corpus).to(DEV)
    with torch.no_grad():
        for prm in model.parameters():
            prm.copy_(torch.randint(-2, 3, prm.shape, generator=torch.Generator().manual_seed(prm.numel())).float())
    ds = plugin.BPRMF.Dataset(model, corpus, "dev")
    runner = BaseRunner(a)
    metrics = runner.evaluate(ds, [1, 10, 100], ["HR", "NDCG"])
    ranks = _device_ranks(runner, ds)
    U = model.u_embeddings.weight.detach().double()
    I = model.i_embeddings.weight.detach().double()
    uid = torch.as_tensor(ev.user_id.values, device=DEV)
    tgt = torch.as_tensor(ev.item_id.values, device=DEV)
    want = np.zeros(rows, np.int64)
    for s in range(0, rows, 64):
        q = U[uid[s:s + 64]]
        S = q @ I.T                                            # [b, n_items]
        s0 = S.gather(1, tgt[s:s + 64, None])
        S[:, 0] = -np.inf
        for r in range(q.shape[0]):
            u = int(ev.user_id[s + r])
            c = torch.as_tensor(sorted(train[u] | residual[u]), device=DEV)
            S[r, c] = -np.inf
        want[s:s + 64] = (1 + (S >= s0).sum(1)).cpu().numpy()
    assert np.array_equal(ranks, want)
    for k in (1, 10, 100):
        assert abs(metrics[f"HR@{k}"] - float((want <= k).mean())) <= 1e-12
        assert abs(metrics[f"NDCG@{k}"] - float(((want <= k) / np.log2(want + 1)).mean())) <= 1e-12


# ---- overlay: the unchanged main.py with and without --device_metrics 1 -------------------------------------------

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
           "--early_stop", "0", "--batch_size", "128", "--eval_batch_size", "50", "--lr", "0.01", "--l2", "0",
           "--topk", "1,5,10", "--model_path", mp, "--log_file", lf, "--regenerate", "1", "--random_seed", "0",
           "--load", str(1 - train), "--train", str(train), "--save_final_results", "0", *flags]
    res = subprocess.run(cmd, cwd=cwd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True,
                         timeout=900)
    out = res.stdout + res.stderr
    assert res.returncode == 0, out[-3000:]
    return re.findall(r"(Test Before Training|Dev  After Training|Test After Training): \(([^)]*)\)", out)


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "main.py")),
                    reason="no unmodified reference staged in oracle/_ref (build() without the checkout)")
@pytest.mark.parametrize("model,flags", [("BPRMF", ["--emb_size", "64"]),
                                         ("BPRMF", ["--emb_size", "64", "--test_all", "1"]),
                                         ("SASRec", ["--emb_size", "32", "--num_heads", "2", "--history_max", "8"])])
def test_overlay_device_metrics_log_the_host_metrics(tmp_path, model, flags):
    tmp = str(tmp_path)
    _dataset(tmp)
    mp = os.path.join(tmp, "model.pt")
    _main(tmp, "train", model, flags, mp, 1)
    host = _main(tmp, "host", model, flags, mp, 0)
    dev = _main(tmp, "dev", model, flags + ["--device_metrics", "1"], mp, 0)
    assert len(host) == 3 and host == dev, (host, dev)
