#!/usr/bin/env python
"""Time of one ``runner.evaluate(dev, ...)`` call on the host route (--device_metrics 0: DataLoader, feed dicts,
collate_batch, predictions copied to the host, evaluate_method) and on the device route (--device_metrics 1: batches
built on the device, ranks and histogram on the device), in one process, alternating the two after a warm-up call of each:

  bprmf_k99          BPRMF d = 64, 1 + 99 candidates, 100k users x 100k items, 20k dev rows
  sasrec_c4          SASRec at bench.py's c4 shape (d = 64, histories up to 50, 2 blocks, 4 heads, 1 M items), 1 + 99
                     candidates, 20k dev rows
  bprmf_test_all_*   BPRMF d = 64 under test_all at 100k and 1M items, 4096 dev rows, 10 train clicks per user.  The host
                     route materialises [rows, n_items] predictions and masks them in a Python loop, so it is timed on a
                     sample of the rows (--buffer 0: feed dicts built per batch; no DataLoader workers, whose
                     [256, n_items] int64 batches would pass through shared memory) and scaled per row; the output says so.
  NeuMF test_all     the fused route against the materialised one at 100k items and the fused route at 1M items
                     (tools/neumf_all_time.py; CUDA events around NeuMF.eval_ranks on one batch of 256 users).

Every other time is a host clock around the evaluate call followed by torch.cuda.synchronize().  The device route's first call
also uploads the phase's columns and builds the clicked-item CSR; it is reported on its own as "first_call_s".  Both routes'
metrics are compared on the rows both evaluated.  One JSON line per case, then one with the card's name, power limit and
max SM clock read in the same run.

    python tools/eval_time.py [--reps 3] [--num_workers 5] [--cases ...]
"""
import argparse
import json
import os
import statistics
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

EVAL_BS = 256
TOPK = [5, 10, 20, 50]
METRICS = ["NDCG", "HR"]


def _clicks(rng, n_users, n_items, per_user):
    return {u: set(rng.randint(1, n_items, per_user).tolist()) for u in range(n_users)}


def _dev_frame(rng, n_users, n_items, rows, K):
    import pandas as pd
    df = pd.DataFrame({"user_id": rng.randint(1, n_users, rows), "item_id": rng.randint(1, n_items, rows),
                       "time": np.arange(rows)})
    if K:
        df["neg_items"] = list(rng.randint(1, n_items, (rows, K)))
    return df


def general_corpus(n_users, n_items, rows, K, seed=0):
    rng = np.random.RandomState(seed)
    dev = _dev_frame(rng, n_users, n_items, rows, K)
    residual = {u: set() for u in range(n_users)}
    for u, i in zip(dev.user_id, dev.item_id):
        residual[int(u)].add(int(i))
    return types.SimpleNamespace(n_users=n_users, n_items=n_items, data_df={"dev": dev},
                                 train_clicked_set=_clicks(rng, n_users, n_items, 10), residual_clicked_set=residual)


def sasrec_corpus(rows, seed=0):
    import ref_arm
    n = 1_000_000
    c = ref_arm.synthetic_corpus(n, n, rows, seed=seed, with_history=50)
    dev = c.data_df["train"]
    dev["neg_items"] = list(np.random.RandomState(seed + 1).randint(1, n, (rows, 99)))
    c.data_df = {"dev": dev}
    return c


CASES = {
    "bprmf_k99": dict(model="BPRMF", flags=["--emb_size", "64"], corpus=lambda: general_corpus(100_000, 100_000, 20_000, 99),
                      test_all=0, host_rows=None),
    "sasrec_c4": dict(model="SASRec", flags=["--emb_size", "64", "--history_max", "50", "--num_layers", "2",
                                             "--num_heads", "4"], corpus=lambda: sasrec_corpus(20_000),
                      test_all=0, host_rows=None),
    "bprmf_test_all_100k": dict(model="BPRMF", flags=["--emb_size", "64"],
                                corpus=lambda: general_corpus(100_000, 100_000, 4096, 0), test_all=1, host_rows=1024),
    "bprmf_test_all_1m": dict(model="BPRMF", flags=["--emb_size", "64"],
                              corpus=lambda: general_corpus(100_000, 1_000_000, 4096, 0), test_all=1, host_rows=256),
}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def run_case(name, reps, num_workers):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    c = CASES[name]
    cls = getattr(plugin, c["model"])
    p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(c["flags"] + ["--test_all", str(c["test_all"]), "--eval_batch_size", str(EVAL_BS),
                                   "--num_workers", str(0 if c["test_all"] else num_workers),
                                   "--buffer", str(0 if c["test_all"] else 1)])
    a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_eval_time.pt", ""
    corpus = c["corpus"]()
    torch.manual_seed(0)
    model = cls(a, corpus).to(a.device)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(20.0)                                   # trained-scale scores
    ds = cls.Dataset(model, corpus, "dev")
    host_ds = ds
    if c["host_rows"]:                                       # the host route on the first host_rows rows
        sub = types.SimpleNamespace(**vars(corpus))
        sub.data_df = {"dev": corpus.data_df["dev"].iloc[:c["host_rows"]]}
        host_ds = cls.Dataset(model, sub, "dev")
    host_ds.prepare()                                        # the reference's buffered feed dicts (when --buffer 1)
    host, dev = BaseRunner(a), BaseRunner(a)
    dev.device_metrics = 1
    t_first, _ = timed(lambda: dev.evaluate(ds, TOPK, METRICS))
    timed(lambda: host.evaluate(host_ds, TOPK, METRICS))     # warm-up
    th, td = [], []
    for _ in range(reps):
        t, m_host = timed(lambda: host.evaluate(host_ds, TOPK, METRICS))
        th.append(t)
        t, m_dev = timed(lambda: dev.evaluate(ds, TOPK, METRICS))
        td.append(t)
    m_dev_same_rows = dev.evaluate(host_ds, TOPK, METRICS) if host_ds is not ds else m_dev
    same = all(abs(m_host[k] - m_dev_same_rows[k]) <= 1e-12 for k in m_host)
    N, Nh = len(ds), len(host_ds)
    h = statistics.median(th)
    out = {"case": name, "rows": N, "n_items": corpus.n_items, "eval_batch_size": EVAL_BS, "reps": reps,
           "device_s": round(statistics.median(td), 4), "device_s_all": [round(x, 4) for x in td],
           "first_call_s": round(t_first, 3), "metrics_equal": same}
    if Nh == N:
        out.update({"host_s": round(h, 4), "host_s_all": [round(x, 4) for x in th]})
    else:
        out.update({"host_rows_measured": Nh, "host_s_measured": round(h, 4), "host_ms_per_row": round(h / Nh * 1e3, 3),
                    "host_s_scaled_to_rows": round(h / Nh * N, 2)})
    out["host_over_device"] = round((out.get("host_s") or out["host_s_scaled_to_rows"]) / out["device_s"], 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--num_workers", type=int, default=5, help="the host route's DataLoader workers (runner default 5)")
    ap.add_argument("--cases", nargs="*", default=list(CASES))
    ap.add_argument("--skip-neumf", action="store_true", help="skip the NeuMF test_all cases")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_time.py measures on a CUDA device; none found")
    from seq_batches_time import card
    for name in a.cases:
        print(json.dumps(run_case(name, a.reps, a.num_workers)), flush=True)
        torch.cuda.empty_cache()
    if not a.skip_neumf:
        from neumf_all_time import neumf_all_items
        for ln in neumf_all_items("ranks", a.reps):
            print(json.dumps(ln), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
