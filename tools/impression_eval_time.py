#!/usr/bin/env python
"""Time of one impression ``evaluate(dev, ...)`` call on the device route (B200ImpressionRunner with --device_metrics 1:
b2r_collate_impression batches, b2r_impression_metrics) and on the host route (the reference's own
ImpressionRunner.evaluate from the copy build() stages in oracle/_ref: DataLoader, one feed dict per impression,
collate_batch, predictions copied to the host, the Python masking loops, evaluate_method), in one process, alternating the
two after a warm-up call of each:

  bprmf    BPRMFImpression, d = 64
  sasrec   SASRecImpression, d = 64, 1 block, 1 head, history_max 20

on 200,000 dev impressions with test_max_pos_item = test_max_neg_item = 20 (lists of 1-25 positives and 1-25 negatives),
eval batch 256, cut-offs 1, 5, 10, 20.  Each time is CUDA events around the call followed by torch.cuda.synchronize().  The
device route's first call also uploads the phase's lists; it is reported on its own as "first_call_s".  The two routes'
metrics are compared (|diff| <= 1e-12).  Without a staged reference only the device route is timed, and the output says so.
One JSON line per case, then one with the card's name, power limit and max SM clock read in the same run.

    python tools/impression_eval_time.py [--reps 3] [--num_workers 5] [--cases bprmf sasrec]
"""
import argparse
import json
import os
import statistics
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
REF = os.path.join(ROOT, "oracle", "_ref", "src")

N_ROWS, N_USERS, N_ITEMS, MP, MN, EVAL_BS, HIS = 200_000, 50_000, 100_000, 20, 20, 256, 30
TOPK = [1, 5, 10, 20]
CASES = {"bprmf": ("BPRMFImpression", ["--emb_size", "64"]),
         "sasrec": ("SASRecImpression", ["--emb_size", "64", "--num_layers", "1", "--num_heads", "1", "--history_max", "20"])}


def corpus(seed=0):
    """a dev phase of N_ROWS impressions as ImpressionReader / ImpressionSeqReader leave it (data_df columns user_id,
    pos_items, neg_items, pos_num, neg_num, position, neg_position) and user_his with HIS positives / 5 negatives per user"""
    import pandas as pd
    rng = np.random.RandomState(seed)
    users = rng.randint(1, N_USERS, N_ROWS)
    npos, nneg = rng.randint(1, MP + 6, N_ROWS), rng.randint(1, MN + 6, N_ROWS)
    flat_p, flat_n = rng.randint(1, N_ITEMS, int(npos.sum())), rng.randint(1, N_ITEMS, int(nneg.sum()))
    pp, np_ = np.concatenate([[0], np.cumsum(npos)]), np.concatenate([[0], np.cumsum(nneg)])
    df = pd.DataFrame({"user_id": users, "pos_items": [flat_p[pp[i]:pp[i + 1]].tolist() for i in range(N_ROWS)],
                       "neg_items": [flat_n[np_[i]:np_[i + 1]].tolist() for i in range(N_ROWS)], "pos_num": npos,
                       "neg_num": nneg, "position": rng.randint(1, HIS + 1, N_ROWS),
                       "neg_position": rng.randint(1, 6, N_ROWS), "time": np.arange(N_ROWS)})
    his_items = rng.randint(1, N_ITEMS, (N_USERS, HIS + 5))
    user_his = {u: {"pos": [(int(i), t) for t, i in enumerate(his_items[u, :HIS])],
                    "neg": [(int(i), t) for t, i in enumerate(his_items[u, HIS:])]} for u in range(N_USERS)}
    return types.SimpleNamespace(n_users=N_USERS, n_items=N_ITEMS, data_df={"dev": df}, user_his=user_his)


def timed(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / 1e3, out


def have_reference() -> bool:
    return os.path.isfile(os.path.join(REF, "main.py"))


def run_case(name, reps, num_workers, c):
    from rechorus_b200 import overlay, plugin
    from rechorus_b200.runner import evaluate_impression_on_device
    cls_name, flags = CASES[name]
    cls = getattr(plugin, cls_name)
    a = cls.parse_model_args(argparse.ArgumentParser()).parse_args(
        flags + ["--test_max_pos_item", str(MP), "--test_max_neg_item", str(MN), "--buffer", "1"])
    a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_imp_time.pt"
    torch.manual_seed(0)
    model = cls(a, c).to(a.device)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(20.0)                                       # trained-scale scores
    out = {"case": name, "model": cls_name, "rows": N_ROWS, "mp": MP, "mn": MN, "eval_batch_size": EVAL_BS,
           "topk": TOPK, "reps": reps}
    if not have_reference():
        data = c.data_df["dev"].to_dict("list")
        if hasattr(model, "history_max"):
            keep = np.asarray(data["position"]) > 0
            data = {k: [v for v, m in zip(col, keep) if m] for k, col in data.items()}
        ds = types.SimpleNamespace(model=model, corpus=c, data=data, phase="dev")
        dev = types.SimpleNamespace(eval_batch_size=EVAL_BS)
        t_first, _ = timed(lambda: evaluate_impression_on_device(dev, ds, TOPK))
        td = [timed(lambda: evaluate_impression_on_device(dev, ds, TOPK))[0] for _ in range(reps)]
        out.update({"device_s": round(statistics.median(td), 4), "device_s_all": [round(x, 4) for x in td],
                    "first_call_s": round(t_first, 3), "host": "not measured: no reference staged in oracle/_ref"})
        return out
    from helpers.ImpressionRunner import ImpressionRunner
    ra = ImpressionRunner.parse_runner_args(argparse.ArgumentParser()).parse_args(
        ["--eval_batch_size", str(EVAL_BS), "--num_workers", str(num_workers)])
    ra.train, ra.log_file = 0, ""
    host = ImpressionRunner(ra)
    ra.device_metrics = 1
    dev = overlay._make_impression_runner_module(ImpressionRunner).B200ImpressionRunner(ra)
    import models.BaseImpressionModel as RI
    ds_cls = RI.ImpressionSeqModel.Dataset if hasattr(model, "history_max") else RI.ImpressionModel.Dataset
    ds = ds_cls(model, c, "dev")
    ds.prepare()                                                  # the reference's buffered feed dicts (--buffer 1)
    metrics = ["NDCG", "HR"]
    t_first, _ = timed(lambda: dev.evaluate(ds, TOPK, metrics))
    timed(lambda: host.evaluate(ds, TOPK, metrics))               # warm-up
    th, td = [], []
    for _ in range(reps):
        t, m_host = timed(lambda: host.evaluate(ds, TOPK, metrics))
        th.append(t)
        t, m_dev = timed(lambda: dev.evaluate(ds, TOPK, metrics))
        td.append(t)
    out.update({"rows": len(ds), "device_s": round(statistics.median(td), 4), "device_s_all": [round(x, 4) for x in td],
                "host_s": round(statistics.median(th), 3), "host_s_all": [round(x, 3) for x in th],
                "first_call_s": round(t_first, 3), "num_workers": num_workers,
                "host_over_device": round(statistics.median(th) / statistics.median(td), 1),
                "same_keys": list(m_host) == list(m_dev),
                "max_abs_diff": max(abs(float(m_host[k]) - float(m_dev[k])) for k in m_host)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--num_workers", type=int, default=5, help="the host route's DataLoader workers (runner default 5)")
    ap.add_argument("--cases", nargs="*", default=list(CASES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("impression_eval_time.py measures on a CUDA device; none found")
    if have_reference():
        for alias, typ in (("object", object), ("int", int), ("float", float)):
            if not hasattr(np, alias):
                setattr(np, alias, typ)                           # removed in NumPy >= 1.24, still used by the reference
        sys.path.insert(0, REF)
    else:
        print("no reference staged in oracle/_ref: timing the device route only", flush=True)
    from seq_batches_time import card
    c = corpus()
    for name in a.cases:
        print(json.dumps(run_case(name, a.reps, a.num_workers, c)), flush=True)
        torch.cuda.empty_cache()
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
