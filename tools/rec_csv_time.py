#!/usr/bin/env python
"""Timings of save_rec_results' CSV write on the device (runner.write_rec_csv, b2r_rec_csv) against the pandas writer,
in one process, on tools/rec_time.py's 100k-user x 100k-item BPRMF test_all corpus (k = 100, eval_batch_size 256):

  runner   BaseRunner.save_rec_results (lists and the device writer) against the pandas route on the same lists (recommend,
           then the DataFrame of Python lists of NumPy scalars and to_csv, as the parent commit wrote it), alternating,
           --reps each; host clocks around calls that end in a device synchronise.  The two files are compared once.
  lists    BaseRunner.recommend alone (the lists and their copy to the host), for scale.
  kernels  the formatting kernels alone (ops.rec_csv over the same lists, in windows of the writer's size): CUDA events
           around all windows, the text's bytes and bytes/s.

One JSON line per measurement, then one with the card's name, power limit and max SM clock read in the same run.

    python tools/rec_csv_time.py [--reps 3] [--out DIR]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def pandas_save(runner, ds, path, k):
    """save_rec_results' pandas route: recommend, then main.py:117-132's DataFrame and to_csv"""
    import pandas as pd
    users, items, scores = runner.recommend(ds, k)
    rec_df = pd.DataFrame(columns=["user_id", "rec_items", "rec_predictions"])
    rec_df["user_id"] = users
    rec_df["rec_items"] = [list(r) for r in items]
    rec_df["rec_predictions"] = [list(r) for r in scores]
    rec_df.to_csv(path, sep="\t", index=False)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for the CSV files (default: a temporary one)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rec_csv_time.py measures on a CUDA device; none found")
    from rec_time import corpus
    from seq_batches_time import card
    from rechorus_b200 import ops, plugin
    from rechorus_b200 import runner as R
    from rechorus_b200.runner import BaseRunner

    k = 100
    p = plugin.BPRMF.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    args = p.parse_args(["--emb_size", "64", "--test_all", "1", "--eval_batch_size", "256", "--num_workers", "0"])
    args.device, args.model_path, args.log_file = torch.device("cuda", 0), "/tmp/_b2r_rec_csv_time.pt", ""
    c = corpus(100_000, 100_000)
    torch.manual_seed(0)
    model = plugin.BPRMF(args, c).to(args.device)
    runner = BaseRunner(args)
    ds = plugin.BPRMF.Dataset(model, c, "test")
    small = corpus(100_000, 100_000)
    small.data_df["test"] = c.data_df["test"].iloc[:500]
    small.train_clicked_set, small.residual_clicked_set = c.train_clicked_set, c.residual_clicked_set
    ds_small = plugin.BPRMF.Dataset(model, small, "test")
    style = R.rec_csv_style("\t", ds.data["user_id"])
    assert style is not None, "NumPy prints in neither style the device writer implements"

    with tempfile.TemporaryDirectory(dir=a.out) as tmp:
        dev_path, pd_path = os.path.join(tmp, "device.csv"), os.path.join(tmp, "pandas.csv")
        runner.save_rec_results(ds_small, dev_path, k)                   # warm-up: modules, shapes, pinned buffers
        pandas_save(runner, ds_small, pd_path, k)
        times = {"device": [], "pandas": []}
        for _ in range(a.reps):
            times["device"].append(timed(lambda: runner.save_rec_results(ds, dev_path, k)))
            times["pandas"].append(timed(lambda: pandas_save(runner, ds, pd_path, k)))
        size = os.path.getsize(dev_path)
        with open(dev_path, "rb") as f1, open(pd_path, "rb") as f2:
            same = f1.read() == f2.read()
        for route in ("device", "pandas"):
            print(json.dumps({"what": f"save_rec_results, {route} writer", "rows": len(ds), "k": k,
                              "s": [round(t, 3) for t in times[route]], "best_s": round(min(times[route]), 3),
                              "file_bytes": size}), flush=True)
        print(json.dumps({"what": "files identical", "value": same}), flush=True)
        lists = [timed(lambda: runner.recommend(ds, k)) for _ in range(a.reps)]
        print(json.dumps({"what": "recommend alone (lists to the host)", "s": [round(t, 3) for t in lists]}), flush=True)

    # the formatting kernels alone, over the same lists, in windows of the writer's size
    users, items, scores = runner.recommend(ds, k)
    du = torch.as_tensor(np.asarray(users, dtype=np.int64)).cuda()
    di, dsc = torch.from_numpy(items).cuda(), torch.from_numpy(scores).cuda()
    kk = items.shape[1]
    row_max = ops.rec_csv_text_bytes_max(1, kk, style)
    W = max(1, R.REC_CSV_WINDOW_BYTES // row_max)
    text = torch.empty(W * row_max, dtype=torch.uint8, device="cuda")
    offs = torch.empty(W + 1, dtype=torch.int64, device="cuda")
    N = du.numel()

    def all_windows():
        total = torch.zeros((), dtype=torch.int64, device="cuda")
        for r0 in range(0, N, W):
            n = min(W, N - r0)
            ops.rec_csv(du[r0:r0 + n], di[r0:r0 + n], dsc[r0:r0 + n], style, "\t", text, offs)
            total += offs[n]
        return total

    all_windows()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.reps):
        e0.record()
        total = all_windows()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        nbytes = int(total)
        print(json.dumps({"what": "formatting kernels (measure, scan, write) over all windows, CUDA events",
                          "rows": N, "k": kk, "window_rows": W, "windows": -(-N // W), "text_bytes": nbytes,
                          "ms": round(ms, 3), "gb_per_s": round(nbytes / ms / 1e6, 1)}), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
