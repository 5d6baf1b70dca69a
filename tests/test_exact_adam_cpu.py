"""CPU: host logic of the exact dense-Adam mode (RowSparseOptimizer(exact_dense=True)) -- which widths it accepts, when
the flush runs, and that every kernel-backed forward hands its ids to the catch-up.  No kernel runs here."""
import argparse
import types

import pytest
import torch


def _model(name, d, extra=()):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(["--emb_size", str(d), "--table_mode", "fused", *extra])
    a.device, a.model_path = torch.device("cpu"), "/tmp/_b2r_exact_cpu.pt"
    return cls(a, types.SimpleNamespace(n_users=20, n_items=30))


@pytest.mark.parametrize("d", [8, 48, 96, 256])
def test_exact_mode_names_a_width_it_has_no_kernel_for(d):
    from rechorus_b200.optim import RowSparseOptimizer
    m = _model("BPRMF", d)
    with pytest.raises(ValueError, match=f"{d} wide"):
        RowSparseOptimizer(m, "Adam", exact_dense=True)
    RowSparseOptimizer(m, "Adam")                            # the lazy mode does not need the catch-up kernel


@pytest.mark.parametrize("d", [32, 64, 128])
def test_exact_mode_accepts_the_catch_up_widths(d):
    from rechorus_b200.optim import RowSparseOptimizer
    opt = RowSparseOptimizer(_model("BPRMF", d), "Adam", exact_dense=True)
    assert all(e["last"].dtype == torch.int32 for e in opt._entries if "last" in e)


def test_flush_runs_once_per_step(monkeypatch):
    from rechorus_b200 import ops
    from rechorus_b200.optim import RowSparseOptimizer
    calls = []
    monkeypatch.setattr(ops, "adam_exact_advance", lambda W, m, v, last, upto, cfg, **kw: calls.append(upto))
    opt = RowSparseOptimizer(_model("BPRMF", 64), "Adam", exact_dense=True)
    opt.flush()
    assert calls == []                                       # nothing stepped yet
    opt.t = 3
    opt.flush()
    opt.flush()
    assert calls == [3, 3]                                   # both tables once; the repeat is skipped
    opt.t = 4
    opt.flush()
    assert calls == [3, 3, 4, 4]


@pytest.mark.parametrize("name,extra,want", [
    ("BPRMF", [], [("u_embeddings.weight", "user_id", -1), ("i_embeddings.weight", "item_id", -1)]),
    ("NeuMF", ["--layers", "[32]"], [("mf_u_embeddings.weight", "user_id", -1), ("mf_i_embeddings.weight", "item_id", -1),
                                     ("mlp_u_embeddings.weight", "user_id", -1),
                                     ("mlp_i_embeddings.weight", "item_id", -1)]),
    ("SASRec", ["--history_max", "5", "--num_layers", "1", "--num_heads", "2"],
     [("i_embeddings.weight", "history_items", 0), ("i_embeddings.weight", "item_id", -1)]),
])
def test_training_forward_catches_up_what_it_reads_and_eval_forward_flushes(name, extra, want, monkeypatch):
    """the forward stops at its first kernel (there is no CPU path); by then the catch-up must have seen every table it
    reads with the ids it reads it with, padding id 0 ignored for SASRec's histories"""
    from rechorus_b200 import ops
    from rechorus_b200.optim import RowSparseOptimizer
    m = _model(name, 32, extra)
    opt = RowSparseOptimizer(m, "Adam", exact_dense=True)
    m.optimizer = opt
    opt.t = 2
    names = {id(p): n for n, p in m.named_parameters()}
    seen, flushes = [], []
    monkeypatch.setattr(opt, "before_forward", lambda p, ids, ignore_id=-1: seen.append((names[id(p)], ids, ignore_id)))
    monkeypatch.setattr(opt, "flush", lambda: flushes.append(opt.t))
    feed = {"user_id": torch.tensor([1, 2]), "item_id": torch.tensor([[3, 4], [5, 6]]), "batch_size": 2,
            "history_items": torch.tensor([[1, 2, 0], [3, 0, 0]]), "lengths": torch.tensor([2, 1])}

    class Stop(Exception):
        pass

    def stop(*a, **k):
        raise Stop()

    for fn in ("embedding", "embed_history"):
        monkeypatch.setattr(ops, fn, stop)
    m.train()
    with pytest.raises(Stop):
        m(feed)
    assert [(n, ig) for n, _, ig in seen] == [(n, ig) for n, _, ig in want]
    for (_, ids, _), (_, key, _) in zip(seen, want):
        assert ids is feed[key]
    assert flushes == []
    seen.clear()
    m.eval()
    with pytest.raises(Stop):
        m(feed)
    assert seen == [] and flushes == [2]
