#!/usr/bin/env python
"""Timings of the top-k recommendation lists (save_rec_results' TopK branch on the device), in one process:

  all_items  ops.topk_all_items(k=100) vs ops.rank_all_items at B = 4096, n_items = 1,000,000, d = 64 (same GEMM tile,
             same fmaf order): CUDA events around each call, mean of --reps after one warm-up call.  FP32 FLOP/s are the
             algorithmic 2 * B * n_items * d over the call time; "share of data-sheet peak" is that rate over the H100 SXM
             data sheet's 67 TFLOP/s FP32 figure.
  rows       ops.topk_rows(k=100) at [65536, 100] and [256, 1,000,000]: CUDA events; bytes/s are the N * C * 4 bytes of
             the prediction matrix read once.
  runner     BaseRunner.save_rec_results (recommend + CSV write) for a 100k-user x 100k-item test_all BPRMF corpus vs the
             reference's host route (predict with the host mask loop, Python sort of every row, CSV write).  The host route
             runs on a 500-user subset and is scaled per row to 100k rows; the output says so.  Host clocks around work
             that ends in a device synchronise.

  split      device time per kernel of one topk_all_items and one rank_all_items call (torch.profiler, CUDA activities),
             in a pass of its own after the timed ones.

One JSON line per measurement, then one with the card's name, power limit and max SM clock read in the same run.

    python tools/rec_time.py [--reps 3] [--skip-runner]
"""
import argparse
import json
import os
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32


def event_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps / 1e3


def random_clicks(rng, n_users, n_items, per_user):
    return {u: set(rng.randint(1, n_items, per_user).tolist()) for u in range(n_users)}


def all_items(reps):
    from rechorus_b200 import ops
    dev = torch.device("cuda", 0)
    B, n_items, d, k = 4096, 1_000_000, 64, 100
    g = torch.Generator(device=dev).manual_seed(0)
    q = torch.randn(B, d, device=dev, generator=g)
    table = torch.randn(n_items, d, device=dev, generator=g)
    rng = np.random.RandomState(0)
    users = np.arange(B, dtype=np.int64)
    target = rng.randint(1, n_items, B).astype(np.int64)
    train = random_clicks(rng, B, n_items, 20)
    residual = {int(u): {int(t)} for u, t in zip(users, target)}
    cs = ops.ClickedSets(train, residual, B, dev)
    mr = np.concatenate([[b] * len(train[b] | residual[b]) for b in range(B)]).astype(np.int64)
    mi = np.concatenate([sorted(train[b] | residual[b]) for b in range(B)]).astype(np.int64)
    tu, tt = torch.from_numpy(users).to(dev), torch.from_numpy(target).to(dev)
    tmr, tmi = torch.from_numpy(mr).to(dev), torch.from_numpy(mi).to(dev)
    flops = 2.0 * B * n_items * d
    out = []
    for name, fn in (("rank_all_items", lambda: ops.rank_all_items(q, table, tt, tmr, tmi)),
                     ("topk_all_items", lambda: ops.topk_all_items(q, table, tt, tu, cs, k)),
                     ("rank_all_items", lambda: ops.rank_all_items(q, table, tt, tmr, tmi)),
                     ("topk_all_items", lambda: ops.topk_all_items(q, table, tt, tu, cs, k))):
        t = event_time(fn, reps)
        out.append({"what": name, "B": B, "n_items": n_items, "d": d, "k": k if "topk" in name else None,
                    "ms": round(t * 1e3, 3), "fp32_tflops": round(flops / t / 1e12, 2),
                    "share_of_datasheet_fp32_peak": round(flops / t / FP32_PEAK, 3)})
    ratio = (out[1]["ms"] + out[3]["ms"]) / (out[0]["ms"] + out[2]["ms"])
    out.append({"what": "topk_all_items / rank_all_items", "ratio": round(ratio, 3)})
    return out


def kernel_split():
    """Device time per kernel of one topk_all_items(k=100) call and one rank_all_items call at the all_items shape, from
    torch.profiler (CUDA activities) in a pass of its own after the timed ones."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from rechorus_b200 import ops
    dev = torch.device("cuda", 0)
    B, n_items, d, k = 4096, 1_000_000, 64, 100
    g = torch.Generator(device=dev).manual_seed(0)
    q = torch.randn(B, d, device=dev, generator=g)
    table = torch.randn(n_items, d, device=dev, generator=g)
    rng = np.random.RandomState(0)
    target = torch.from_numpy(rng.randint(1, n_items, B).astype(np.int64)).to(dev)
    users = torch.arange(B, dtype=torch.int64, device=dev)
    cs = ops.ClickedSets(random_clicks(rng, B, n_items, 20), {}, B, dev)
    out = []
    for name, fn in (("topk_all_items", lambda: ops.topk_all_items(q, table, target, users, cs, k)),
                     ("rank_all_items", lambda: ops.rank_all_items(q, table, target))):
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        per = {}
        for ev in prof.events():
            if ev.device_type != DeviceType.CUDA or "b2r::" not in ev.name:
                continue
            key = ev.name.split("(")[0].replace("void ", "")
            c, tot = per.get(key, (0, 0.0))
            per[key] = (c + 1, tot + ev.device_time_total)              # microseconds
        total = sum(v[1] for v in per.values())
        out.append({"what": "kernel split of one " + name + " call (torch.profiler)",
                    "total_kernel_ms": round(total / 1e3, 3),
                    "kernels": {kname: {"launches": c, "ms": round(t / 1e3, 3), "share": round(t / total, 3)}
                                for kname, (c, t) in sorted(per.items(), key=lambda kv: -kv[1][1])}})
    return out


def rows(reps):
    from rechorus_b200 import ops
    dev = torch.device("cuda", 0)
    out = []
    for N, C in ((65536, 100), (256, 1_000_000)):
        x = torch.randn(N, C, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
        t = event_time(lambda: ops.topk_rows(x, 100), reps)
        out.append({"what": "topk_rows", "N": N, "C": C, "k": 100, "ms": round(t * 1e3, 3),
                    "gb_per_s": round(N * C * 4 / t / 1e9, 1)})
    return out


def corpus(n_users, n_items, seed=0):
    import pandas as pd
    rng = np.random.RandomState(seed)
    users = np.arange(1, n_users)
    test = pd.DataFrame({"user_id": users, "item_id": rng.randint(1, n_items, len(users)), "time": 0})
    train = random_clicks(rng, n_users, n_items, 10)
    residual = {int(u): {int(i)} for u, i in zip(test.user_id, test.item_id)}
    residual[0] = set()
    return types.SimpleNamespace(n_users=n_users, n_items=n_items, data_df={"train": test, "dev": test, "test": test},
                                 train_clicked_set=train, residual_clicked_set=residual)


def runner_route():
    import pandas as pd
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    n_users = n_items = 100_000
    p = plugin.BPRMF.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(["--emb_size", "64", "--test_all", "1", "--eval_batch_size", "256", "--num_workers", "0"])
    a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_rec_time.pt", ""
    c = corpus(n_users, n_items)
    torch.manual_seed(0)
    model = plugin.BPRMF(a, c).to(a.device)
    runner = BaseRunner(a)
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        ds = plugin.BPRMF.Dataset(model, c, "test")
        small = corpus(n_users, n_items)
        small.data_df["test"] = c.data_df["test"].iloc[:500]
        small.train_clicked_set, small.residual_clicked_set = c.train_clicked_set, c.residual_clicked_set
        ds_small = plugin.BPRMF.Dataset(model, small, "test")
        ds_small.prepare()                                                        # the reference's buffered feed dicts
        runner.save_rec_results(ds_small, os.path.join(tmp, "warm.csv"))          # warm-up (module load, shapes)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        users, items, scores = runner.recommend(ds, 100)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        runner.save_rec_results(ds, os.path.join(tmp, "dev.csv"))
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        out.append({"what": "device route", "rows": len(ds), "recommend_s": round(t1 - t0, 3),
                    "recommend_plus_csv_s": round(t2 - t1, 3)})
        # the reference's route (main.py:117-132 + BaseRunner.py:225-252) on 500 rows
        t0 = time.perf_counter()
        preds = runner.predict(ds_small)
        rec_items, rec_preds = [], []
        for i in range(len(ds_small)):
            info = ds_small[i]
            lst = sorted(zip(info["item_id"], preds[i]), key=lambda x: x[1], reverse=True)[:100]
            rec_items.append([x[0] for x in lst])
            rec_preds.append([x[1] for x in lst])
        df = pd.DataFrame(columns=["user_id", "rec_items", "rec_predictions"])
        df["user_id"] = list(ds_small.data["user_id"])
        df["rec_items"], df["rec_predictions"] = rec_items, rec_preds
        df.to_csv(os.path.join(tmp, "host.csv"), sep="\t", index=False)
        t = time.perf_counter() - t0
        out.append({"what": "host route (measured on a 500-user subset, scaled per row)", "rows_measured": 500,
                    "ms_per_row": round(t / 500 * 1e3, 3), "scaled_to_rows": len(ds),
                    "scaled_s": round(t / 500 * len(ds), 1)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skip-runner", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rec_time.py measures on a CUDA device; none found")
    from seq_batches_time import card
    for part in (all_items, rows) + (() if a.skip_runner else (runner_route,)) + (kernel_split,):
        for ln in part(a.reps) if part in (all_items, rows) else part():
            print(json.dumps(ln), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
