#!/usr/bin/env python
"""What the exact dense-Adam mode (--exact_adam 1) costs, on one GPU, in one process, the variants alternated:

  c2      BPRMF 1M x 1M, d = 64, B = 4096, C = 100: the single-call step (model.train_step, next batch prefetched),
          lazy row-sparse Adam against the exact mode; CUDA events around `--steps` steps, per round
  c3, c4  NeuMF (4 tables of 1M x 64, layers [64, 32, 16], C = 5) and SASRec (1M items, L = 50, 2 blocks, 4 heads,
          C = 100) at B = 4096 on device-built batches (--device_batches, eager contract step): one epoch per round per
          variant, host clock around runner.fit + synchronize, after one untimed warm-up epoch each:
            lazy   fused tables, row-sparse Adam (untouched rows do not move)
            exact  fused tables, --exact_adam 1 (dense torch.optim.Adam results)
            dense  dense tables and the optimizer's dense torch-formula Adam over every row (b2r_dense_optim)

Adam lr = 1e-3 with l2 = 1e-6, the weight decay of the documented BPRMF / SASRec command lines.  One JSON line per
(config, variant) with every round's time and the median, then one with the card's name, power limit and max SM clock
read in the same run.

    python tools/exact_adam_time.py [--rounds 5] [--steps 20] [--batches 8] [--configs c2 c3 c4]
"""
import argparse
import gc
import json
import os
import statistics
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

N, B, LR, L2 = 1_000_000, 4096, 1e-3, 1e-6
MODELS = {
    "c3": ("NeuMF", ["--emb_size", "64", "--layers", "[64, 32, 16]", "--num_neg", "4"], 0),
    "c4": ("SASRec", ["--emb_size", "64", "--history_max", "50", "--num_layers", "2", "--num_heads", "4",
                      "--num_neg", "99"], 50),
}


def card():
    from seq_batches_time import card as _card
    return _card()


def c2(rounds, steps):
    from rechorus_b200 import plugin
    from rechorus_b200.optim import RowSparseOptimizer
    from rechorus_b200.runner import BaseRunner
    dev = torch.device("cuda", 0)
    C = 100

    def model(exact):
        p = plugin.BPRMF.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
        a = p.parse_args(["--emb_size", "64", "--num_neg", str(C - 1), "--table_mode", "fused"])
        a.device, a.model_path = dev, "/tmp/_b2r_exact_time.pt"
        torch.manual_seed(0)
        m = plugin.BPRMF(a, types.SimpleNamespace(n_users=N, n_items=N)).to(dev)
        m.optimizer = RowSparseOptimizer(m, "Adam", lr=LR, l2=L2, exact_dense=exact)
        m.train()
        return m

    g = torch.Generator().manual_seed(3)
    feeds = [{"user_id": torch.randint(1, N, (B,), generator=g).to(dev),
              "item_id": torch.randint(1, N, (B, C), generator=g).to(dev), "batch_size": B, "phase": "train"}
             for _ in range(8)]
    models = {"lazy": model(False), "exact": model(True)}

    def run(m, n):
        for k in range(n):
            m.train_step(feeds[k % len(feeds)], feeds[(k + 1) % len(feeds)] if k + 1 < n else None)

    for m in models.values():
        run(m, 10)                                           # warm-up: contexts, modules, plans
    torch.cuda.synchronize()
    ms = {v: [] for v in models}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for v, m in models.items():
            ev0.record()
            run(m, steps)
            ev1.record()
            ev1.synchronize()
            ms[v].append(ev0.elapsed_time(ev1) / steps)
    for v, xs in ms.items():
        print(json.dumps({"config": "c2", "route": "single-call step (train_step)", "variant": v, "B": B, "C": C,
                          "ms_per_step": [round(x, 4) for x in xs], "median_ms_per_step": round(statistics.median(xs), 4),
                          "t": models[v].optimizer.t}), flush=True)
    del models
    gc.collect()
    torch.cuda.empty_cache()


def model_epochs(cfg, rounds, batches):
    import ref_arm
    from rechorus_b200 import plugin
    from rechorus_b200.optim import RowSparseOptimizer
    from rechorus_b200.runner import BaseRunner
    name, flags, hist = MODELS[cfg]
    cls = getattr(plugin, name)
    corpus = ref_arm.synthetic_corpus(N, N, batches * B, seed=0, with_history=hist)
    arms = {}
    for v in ("lazy", "exact", "dense"):
        p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
        fl = flags + ["--batch_size", str(B), "--num_workers", "0", "--lr", str(LR), "--l2", str(L2), "--optimizer",
                      "Adam", "--device_batches", "7"]
        if v != "dense":
            fl += ["--table_mode", "fused", "--fused_optimizer", "1", "--exact_adam", str(int(v == "exact"))]
        a = p.parse_args(fl)
        a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_exact_time.pt", ""
        torch.manual_seed(0)
        m = cls(a, corpus).to(a.device)
        if v == "dense":
            m.optimizer = RowSparseOptimizer(m, "Adam", lr=LR, l2=L2)         # tables stay dense: b2r_dense_optim
        runner = BaseRunner(a)
        data = cls.Dataset(m, corpus, "train")
        runner.fit(data, epoch=0)                                              # warm-up epoch
        arms[v] = (m, runner, data)
    torch.cuda.synchronize()
    secs = {v: [] for v in arms}
    losses = {v: [] for v in arms}
    for r in range(rounds):
        for v, (m, runner, data) in arms.items():
            t0 = time.perf_counter()
            losses[v].append(runner.fit(data, epoch=r + 1))
            torch.cuda.synchronize()
            secs[v].append(time.perf_counter() - t0)
    for v, xs in secs.items():
        ms = [1e3 * x / batches for x in xs]
        print(json.dumps({"config": cfg, "model": name, "route": "device batches, eager contract step", "variant": v,
                          "B": B, "steps_per_epoch": batches, "ms_per_step": [round(x, 3) for x in ms],
                          "median_ms_per_step": round(statistics.median(ms), 3), "losses": losses[v],
                          "t": arms[v][0].optimizer.t}), flush=True)
    del arms
    gc.collect()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20, help="c2: timed single-call steps per round")
    ap.add_argument("--batches", type=int, default=8, help="c3 / c4: full-size batches per epoch")
    ap.add_argument("--configs", nargs="+", default=["c2", "c3", "c4"])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("exact_adam_time.py measures on a CUDA device; none is visible")
    for cfg in a.configs:
        if cfg == "c2":
            c2(a.rounds, a.steps)
        else:
            model_epochs(cfg, a.rounds, a.batches)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
