"""NeuMF under test_all (d = 64, layers [64, 32, 16], one evaluation batch, 20 clicked items per user):
the fused route (ops.neumf_score_rows window by window, then the mask / rank / top-k kernels) against the materialised
route (NeuMF.forward on the [Bn * n_items] candidate matrix, then the same kernels).  Used by tools/eval_time.py (kind
"ranks": NeuMF.eval_ranks) and tools/rec_time.py (kind "lists": NeuMF.recommend, k = 100).

  100k items  both routes, alternating, --reps calls each after a warm-up call, on a batch of 40 users: the materialised
              route cannot run the default eval batch of 256 there, because its output layer's SGEMM launches one row of
              CTAs per 64 candidate rows and the grid stops at 65535 rows (4.19M candidates, 41 users).  CUDA events around
              each call, the mean, and the peak of torch.cuda.max_memory_allocated above the inputs during that route's
              calls.  The fused route is also timed alone on a batch of 256.
  1M items    a batch of 256, the fused route only (the materialised one would need a 131 GB concat buffer).  Two
              per-row samples, each scaled to the 256 rows: the materialised device route on single rows (a one-row
              forward, then the same kernels; CUDA events), and the host route (BaseRunner.predict's forward and copy to
              the host, its Python mask loop over the clicked items, then BaseRunner's rank for "ranks" or main.py's
              sorted(zip(item_id, prediction))[:100] for "lists"; a host clock ending in a device synchronise).
"""
import time

import numpy as np
import torch

D, LAYERS, BN, BN_BOTH, K = 64, [64, 32, 16], 256, 40, 100


def _setup(n_items, Bn, n_users=1000):
    import argparse
    import types
    from rechorus_b200 import ops, plugin
    p = plugin.NeuMF.parse_model_args(argparse.ArgumentParser())
    a = p.parse_args(["--emb_size", str(D), "--layers", str(LAYERS), "--test_all", "1"])
    a.device, a.model_path = torch.device("cuda", 0), ""
    torch.manual_seed(0)
    m = plugin.NeuMF(a, types.SimpleNamespace(n_users=n_users, n_items=n_items)).to(a.device)
    with torch.no_grad():
        for prm in m.parameters():
            prm.mul_(20.0)
    m.eval()
    rng = np.random.RandomState(0)
    users = torch.from_numpy(rng.randint(0, n_users, Bn).astype(np.int64)).to(a.device)
    ids = torch.arange(n_items, dtype=torch.int64, device=a.device).repeat(Bn, 1)
    ids[:, 0] = torch.from_numpy(rng.randint(1, n_items, Bn).astype(np.int64)).to(a.device)
    clicked = {u: set(rng.randint(1, n_items, 20).tolist()) for u in range(n_users)}
    cs = ops.ClickedSets(clicked, {}, n_users, a.device)
    return m, {"user_id": users, "item_id": ids, "batch_size": Bn, "phase": "test"}, cs


def _routes(m, kind):
    from rechorus_b200 import plugin
    base = plugin._KernelModelMixin                 # the materialised route: the mixin's forward-based methods
    if kind == "ranks":
        return (lambda f, c: m.eval_ranks(f, clicked=c)), (lambda f, c: base.eval_ranks(m, f, clicked=c))
    return (lambda f, c: m.recommend(f, K, c)), (lambda f, c: base.recommend(m, f, K, c))


def _timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, torch.cuda.max_memory_allocated() - base


def neumf_all_items(kind, reps):
    out = []
    m, feed, cs = _setup(100_000, BN_BOTH)
    fused, mat = _routes(m, kind)
    fused(feed, cs), mat(feed, cs)                  # warm-up
    ms = {"fused": [], "materialised": []}
    peak = {"fused": 0, "materialised": 0}
    for _ in range(reps):
        for name, fn in (("materialised", mat), ("fused", fused)):
            t, p = _timed(lambda: fn(feed, cs), 1)
            ms[name].append(t)
            peak[name] = max(peak[name], p)
    for name in ("materialised", "fused"):
        out.append({"what": f"NeuMF test_all {kind}, {name} route", "n_items": 100_000, "Bn": BN_BOTH, "d": D,
                    "layers": LAYERS, "ms": round(float(np.mean(ms[name])), 3),
                    "ms_each": [round(x, 3) for x in ms[name]], "peak_mib_above_inputs": round(peak[name] / 2 ** 20, 1)})
    out.append({"what": f"NeuMF test_all {kind} at 100k items: materialised / fused",
                "ratio": round(float(np.mean(ms["materialised"]) / np.mean(ms["fused"])), 2)})
    del m, feed, cs, fused, mat
    torch.cuda.empty_cache()

    for n_items in (100_000, 1_000_000):
        m, feed, cs = _setup(n_items, BN)
        fused, mat = _routes(m, kind)
        fused(feed, cs)
        t, p = _timed(lambda: fused(feed, cs), reps)
        out.append({"what": f"NeuMF test_all {kind}, fused route", "n_items": n_items, "Bn": BN, "d": D,
                    "layers": LAYERS, "ms": round(t, 3), "peak_mib_above_inputs": round(p / 2 ** 20, 1)})
        if n_items == 100_000:
            del m, feed, cs, fused, mat
            torch.cuda.empty_cache()
    rows = 4
    one = lambda b: {"user_id": feed["user_id"][b:b + 1], "item_id": feed["item_id"][b:b + 1], "batch_size": 1}
    mat(one(0), cs)
    t, p = _timed(lambda: [mat(one(b), cs) for b in range(rows)], 1)
    out.append({"what": f"NeuMF test_all {kind}, materialised route (measured on {rows} single rows, scaled per row)",
                "n_items": 1_000_000, "ms_per_row": round(t / rows, 3), "scaled_to_rows": BN,
                "scaled_ms": round(t / rows * BN, 1), "peak_mib_above_inputs_one_row": round(p / 2 ** 20, 1)})
    host_rows = 2
    ids_host = np.arange(m.item_num)
    masks = [clicked_of(cs, int(feed["user_id"][b])) for b in range(host_rows)]    # the host's clicked sets
    targets = [int(feed["item_id"][b, 0]) for b in range(host_rows)]
    with torch.no_grad():
        m.forward(one(0))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for b in range(host_rows):
            ids_host[0] = targets[b]
            pred = m.forward(one(b))["prediction"].cpu().numpy()[0]
            for it in masks[b]:                                       # BaseRunner.py:244-251
                pred[it] = -np.inf
            if kind == "ranks":
                int((pred >= pred[0]).sum())                          # BaseRunner.py:63
            else:
                sorted(zip(ids_host, pred), key=lambda x: x[1], reverse=True)[:K]    # main.py:121-126
        t = (time.perf_counter() - t0) * 1e3
    out.append({"what": f"NeuMF test_all {kind}, host route (measured on {host_rows} rows, scaled per row)",
                "n_items": 1_000_000, "ms_per_row": round(t / host_rows, 1), "scaled_to_rows": BN,
                "scaled_s": round(t / host_rows * BN / 1e3, 1)})
    del m, feed, cs, fused, mat
    torch.cuda.empty_cache()
    return out


def clicked_of(cs, u):
    """user u's clicked items from the device CSR, as the host-side set BaseRunner masks"""
    lo, hi = int(cs.ptr[u]), int(cs.ptr[u + 1])
    return cs.items[lo:hi].cpu().tolist()
