#!/usr/bin/env python
"""Whole SASRec training epochs at bench.py's c4 shape (B = 4096, K = 99, histories up to 50, 2 blocks, 4 heads, d = 64,
fused Adam) on three batch-production routes, in one process:

  host    runner.fit on the host data path (SequentialModel.Dataset feed dicts, collate_batch, DataLoader, NumPy negatives)
  device  --device_batches: negatives, row shuffle and collate (histories included) as device kernels, eager steps
  graph   --device_batches with --graph_step 1: the same batches, full-size steps replayed as one CUDA graph

Each route gets a fresh, identically initialised model, one untimed warm-up epoch, then `--epochs` timed epochs: host
clocks around ``runner.fit`` followed by ``torch.cuda.synchronize()``.  One JSON line per route, then one with the card's
name, power limit and max SM clock read in the same run.

    python tools/seq_batches_time.py [--batches 16] [--epochs 1]
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N = 1_000_000
B = 4096
L = 50
MODEL = ["--emb_size", "64", "--history_max", str(L), "--num_layers", "2", "--num_heads", "4", "--num_neg", "99"]
ROUTES = {"host": [], "device": ["--device_batches", "7"], "graph": ["--device_batches", "7", "--graph_step", "1"]}


def card():
    dev = torch.device("cuda", 0)
    out = {"gpu": torch.cuda.get_device_name(dev)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        pl, clk = [x.strip() for x in q.strip().splitlines()[0].split(",")]
        out["power_limit_w"], out["sm_max_mhz"] = float(pl), int(float(clk))
    except Exception as e:                                   # the query is informational; the times stand without it
        out["nvidia_smi"] = repr(e)[:200]
    return out


def run(route, corpus, epochs):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    p = plugin.SASRec.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(MODEL + ["--batch_size", str(B), "--num_workers", "0", "--lr", "1e-3", "--optimizer", "Adam",
                              "--table_mode", "fused", "--fused_optimizer", "1"] + ROUTES[route])
    a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_seq_batches.pt", ""
    torch.manual_seed(0)
    model = plugin.SASRec(a, corpus).to(a.device)
    data = plugin.SASRec.Dataset(model, corpus, "train")
    runner = BaseRunner(a)
    warm = runner.fit(data, epoch=0)
    torch.cuda.synchronize()
    times, losses = [], []
    for e in range(epochs):
        t0 = time.perf_counter()
        losses.append(runner.fit(data, epoch=e + 1))
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    steps = (len(data) + B - 1) // B
    s = sum(times) / len(times)
    return {"route": route, "rows": len(data), "steps_per_epoch": steps, "s_per_epoch": round(s, 4),
            "ms_per_step": round(1e3 * s / steps, 3), "warmup_loss": warm, "losses": losses,
            "graphed": "_b2r_graphed_step" in model.__dict__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=16, help="full-size batches per epoch (a ragged one is added)")
    ap.add_argument("--epochs", type=int, default=1)
    ap.add_argument("--routes", nargs="+", default=list(ROUTES))
    a = ap.parse_args()
    import ref_arm
    corpus = ref_arm.synthetic_corpus(N, N, a.batches * B + B // 2, seed=0, with_history=L)
    for route in a.routes:
        print(json.dumps(run(route, corpus, a.epochs)), flush=True)
        gc.collect()                                         # the captured step and the model refer to each other
        torch.cuda.empty_cache()
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
