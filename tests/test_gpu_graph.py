"""GPU: a whole contract-route training step captured in a CUDA graph (rechorus_b200.graph.GraphedStep) must train exactly
like the same steps launched eagerly: the device-side optimizer clock (b2r_optim_tick) replaces the per-step host
parameters (Adam's bias corrections), everything else is the same kernels in the same order."""
import argparse
import types

import pytest
import torch

pytestmark = pytest.mark.gpu


def _build(name, flags, device_clock):
    from rechorus_b200 import plugin
    from rechorus_b200.optim import RowSparseOptimizer
    cls = getattr(plugin, name)
    p = cls.parse_model_args(argparse.ArgumentParser())
    a = p.parse_args(flags + ["--table_mode", "fused"])
    a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_graph.pt"
    torch.manual_seed(3)
    m = cls(a, types.SimpleNamespace(n_users=200, n_items=300)).to(a.device)
    with torch.no_grad():
        for q in m.parameters():
            q.mul_(10.0)
    m.optimizer = RowSparseOptimizer(m, "Adam", lr=1e-2, l2=1e-5, eps=1e-3, device_clock=device_clock)
    m.train()
    return m


def _feeds(name, n, B=64, C=6, L=9):
    g = torch.Generator().manual_seed(8)
    out = []
    for _ in range(n):
        f = {"user_id": torch.randint(1, 200, (B,), generator=g).cuda(), "item_id": torch.randint(1, 300, (B, C), generator=g).cuda(),
             "batch_size": B, "phase": "train"}
        if name == "SASRec":
            lengths = torch.randint(1, L + 1, (B,), generator=g)
            lengths[0] = L
            f["history_items"] = (torch.randint(1, 300, (B, L), generator=g) * (torch.arange(L).view(1, L) < lengths.view(B, 1))).cuda()
            f["lengths"] = lengths.cuda()
        out.append(f)
    return out


@pytest.mark.parametrize("name,flags", [("BPRMF", ["--emb_size", "64"]),
                                        ("NeuMF", ["--emb_size", "32", "--layers", "[32, 16]"]),
                                        ("SASRec", ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "9"])])
def test_graphed_steps_equal_eager_steps(name, flags):
    from rechorus_b200 import ops
    from rechorus_b200.graph import GraphedStep
    feeds = _feeds(name, 7)
    eager = _build(name, flags, device_clock=False)
    graphed = _build(name, flags, device_clock=True)
    step = GraphedStep(graphed, feeds[0], warmup=2)          # 2 eager warm-up steps on feeds[0], then the capture
    losses_e = []
    for f in [feeds[0], feeds[0]] + feeds[1:]:               # the same sequence of batches, eagerly
        eager.optimizer.zero_grad()
        ls = eager.loss(eager(f))
        ls.backward()
        eager.optimizer.step()
        losses_e.append(float(ls))
    losses_g = [float(step(f)) for f in feeds[1:]]
    torch.cuda.synchronize()
    assert graphed.optimizer.sync_clock() == eager.optimizer.t == 8
    # the device clock reproduces the host route's float32 bias corrections: same step sizes, same kernels, same order
    tol_l, tol_w = 1e-6 * max(1.0, max(losses_e)), 1e-6
    for a, b in zip(losses_g, losses_e[2:]):
        assert abs(a - b) <= tol_l, (losses_g, losses_e)
    for (k, pa), (_, pb) in zip(graphed.named_parameters(), eager.named_parameters()):
        assert (pa - pb).abs().max() <= tol_w, k
    ops.check_ids()


def test_capture_after_eager_steps_on_the_default_stream():
    """the runner's natural order: some eager steps (default stream, ``loss.backward()``, losses not kept) and THEN the
    capture; eager steps keep working afterwards (the ragged last batch of an epoch)."""
    from rechorus_b200.graph import GraphedStep
    name, flags = "NeuMF", ["--emb_size", "32", "--layers", "[32, 16]"]
    feeds = _feeds(name, 4)
    m = _build(name, flags, device_clock=True)
    for f in feeds[:2]:
        m.optimizer.zero_grad()
        m.loss(m(f)).backward()
        m.optimizer.step()
    step = GraphedStep(m, feeds[2], warmup=1)
    l1 = float(step(feeds[3]))
    l2 = float(step(feeds[3]))
    assert l2 < l1 and m.optimizer.sync_clock() == 2 + 1 + 2
    m.optimizer.zero_grad()                                   # and eager steps keep working after the capture
    m.loss(m(feeds[0])).backward()
    m.optimizer.step()
    torch.cuda.synchronize()


@pytest.mark.parametrize("model_name,extra", [("NeuMF", ["--emb_size", "32", "--layers", "[32]"])])
def test_runner_graph_step_trains_like_the_eager_loop(model_name, extra):
    """--graph_step 1: BaseRunner.fit replays the captured loop body for the full-size batches (the first one trains through
    the capture's warm-up step, the ragged last one eagerly); two epochs must end where the eager loop ends (which also
    applies the reference's candidate shuffle -- a no-op up to summation order)"""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import fit_corpus
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, model_name)

    def run(graph):
        p = argparse.ArgumentParser()
        p = BaseRunner.parse_runner_args(p)
        p = cls.parse_model_args(p)
        a = p.parse_args(extra + ["--num_neg", "5", "--batch_size", "64", "--num_workers", "0", "--lr", "0.001", "--optimizer",
                                  "Adam", "--table_mode", "fused", "--fused_optimizer", "1", "--graph_step", str(graph)])
        a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_gs.pt", ""
        corpus = fit_corpus.build()
        torch.manual_seed(1)
        import numpy as np
        np.random.seed(1)
        model = cls(a, corpus).to(a.device)
        train = cls.Dataset(model, corpus, "train")
        runner = BaseRunner(a)
        ls = [runner.fit(train, epoch=e) for e in (1, 2)]
        torch.cuda.synchronize()
        return model, ls, runner

    m0, l0, _ = run(0)
    m1, l1, r1 = run(1)
    assert "_b2r_graphed_step" in m1.__dict__ and m1.optimizer.t == m0.optimizer.t
    for a, b in zip(l0, l1):
        assert abs(a - b) <= 1e-4, (l0, l1)
    # the two loops differ in summation order only (the eager one scores shuffled columns); Adam turns a 1e-10 difference
    # of a gradient entry that is within a few orders of eps into a visible fraction of lr (DESIGN.md section 6), so the
    # bulk is bounded tightly and the ill-conditioned tail by the 12 steps' worth of lr = 1e-3 it can drift at most
    for (k, pa), (_, pb) in zip(m0.named_parameters(), m1.named_parameters()):
        d = (pa.detach() - pb.detach()).abs().flatten()
        assert float(d.median()) <= 1e-6 and float(d.max()) <= 2e-2, (k, float(d.median()), float(d.max()))
