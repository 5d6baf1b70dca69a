#!/usr/bin/env python
"""Training-step time of the c3 (NeuMF) and c4 (SASRec) shapes of bench.py with and without dropout, on the eager route
(forward, loss, backward and optimizer step launched from Python) and replayed as a CUDA graph (rechorus_b200.graph).
CUDA events around `--steps` steps after `--warmup` warm-up steps; one JSON line per (model, p, route).  A route that
cannot run in this tree is reported with its error instead of a time.

    python tools/dropout_time.py [--steps 50] [--warmup 10] [--p 0 0.2] [--models c3 c4]
"""
import argparse
import json
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

N = 1_000_000
B = 4096
L = 50
SHAPES = {"c3": ("NeuMF", ["--emb_size", "64", "--layers", "[64, 32, 16]", "--num_neg", "4"], 5),
          "c4": ("SASRec", ["--emb_size", "64", "--history_max", "50", "--num_layers", "2", "--num_heads", "4",
                            "--num_neg", "99"], 100)}


def build(name, extra, p, graph, dev):
    from rechorus_b200 import plugin
    from rechorus_b200.optim import RowSparseOptimizer
    cls = getattr(plugin, name)
    a = cls.parse_model_args(argparse.ArgumentParser()).parse_args(extra + ["--table_mode", "fused", "--dropout", str(p)])
    a.device, a.model_path = dev, "/tmp/_b2r_unused.pt"
    torch.manual_seed(0)
    m = cls(a, types.SimpleNamespace(n_users=N, n_items=N)).to(dev)
    m.optimizer = RowSparseOptimizer(m, "Adam", lr=1e-3, device_clock=graph)
    m.train()
    return m


def feeds(name, C, dev):
    g = torch.Generator().manual_seed(0)
    out = []
    for _ in range(4):
        f = {"user_id": torch.randint(1, N, (B,), generator=g).to(dev), "item_id": torch.randint(1, N, (B, C), generator=g).to(dev),
             "batch_size": B, "phase": "train"}
        if name == "SASRec":
            lengths = torch.randint(1, L + 1, (B,), generator=g)
            lengths[0] = L
            f["history_items"] = (torch.randint(1, N, (B, L), generator=g) * (torch.arange(L).view(1, L) < lengths.view(B, 1))).to(dev)
            f["lengths"] = lengths.to(dev)
        out.append(f)
    return out


def time_route(m, fs, graph, steps, warmup):
    if graph:
        from rechorus_b200.graph import GraphedStep
        gs = GraphedStep(m, fs[0], warmup=2)
        step = lambda k: gs(fs[k % len(fs)])                         # noqa: E731
    else:
        def step(k):
            m.optimizer.zero_grad()
            loss = m.loss(m(fs[k % len(fs)]))
            loss.backward()
            m.optimizer.step()
            return loss.detach()
    for k in range(warmup):
        step(k)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(steps):
        loss = step(k)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, float(loss)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--p", type=float, nargs="+", default=[0.0, 0.2])
    ap.add_argument("--models", nargs="+", default=["c3", "c4"])
    ap.add_argument("--tag", default="")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    gpu = torch.cuda.get_device_name(dev)
    for key in a.models:
        name, extra, C = SHAPES[key]
        fs = feeds(name, C, dev)
        for p in a.p:
            for graph in (False, True):
                rec = {"tag": a.tag, "workload": key, "model": name, "p": p, "route": "graph" if graph else "eager", "gpu": gpu}
                try:
                    m = build(name, extra, p, graph, dev)
                    rec["ms_per_step"], rec["loss"] = time_route(m, fs, graph, a.steps, a.warmup)
                except Exception as e:                          # e.g. a tree whose graphed step cannot capture this model
                    rec["error"] = repr(e)[:300]
                print(json.dumps(rec), flush=True)
                m = None
                torch.cuda.synchronize()
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
