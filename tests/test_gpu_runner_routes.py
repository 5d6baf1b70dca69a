"""GPU: the runner's training routes where they must agree with each other -- the CPU random streams every host route
draws (reference fit, --fused_step 1, --graph_step 1), a --fused_step epoch against the same DataLoader batches stepped by
hand, and when the graph route captures, replays and steps eagerly, on host batches (SASRec, padded to each batch's own
width) and on device batches (fit_on_device, full batches collated straight into the captured inputs)."""
import argparse
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BPRMF = ["--emb_size", "64", "--num_neg", "3"]
SASREC = ["--emb_size", "32", "--num_layers", "1", "--num_heads", "2", "--history_max", "16", "--num_neg", "3"]
NEUMF = ["--emb_size", "32", "--layers", "[32, 16]", "--num_neg", "5"]


def _setup(model_name, flags, seed=1):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import fit_corpus
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, model_name)
    p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(["--batch_size", "64", "--num_workers", "0", "--lr", "0.01", "--optimizer", "Adam",
                      "--table_mode", "fused", "--fused_optimizer", "1"] + flags)
    a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_routes.pt", ""
    corpus = fit_corpus.build()
    torch.manual_seed(seed)
    np.random.seed(seed)
    model = cls(a, corpus).to(a.device)
    return model, cls.Dataset(model, corpus, "train"), BaseRunner(a)


def _shapes(feed):
    return {k: tuple(v.shape) for k, v in feed.items() if isinstance(v, torch.Tensor)}


def _record_graph_steps(monkeypatch, model):
    """one (kind, shapes) event per training step: "capture" (GraphedStep.__init__, whose warm-up step trains the batch),
    "call" (GraphedStep.__call__: copy in, replay), "replay" (GraphedStep.replay on inputs written in place) or "eager"
    (a forward outside a capture)"""
    from rechorus_b200 import graph
    events, capturing = [], [False]
    init, call, replay = graph.GraphedStep.__init__, graph.GraphedStep.__call__, graph.GraphedStep.replay

    def counting_init(self, m, feed, warmup=2):
        events.append(("capture", _shapes(feed)))
        capturing[0] = True
        try:
            init(self, m, feed, warmup)
        finally:
            capturing[0] = False

    def counting_call(self, feed):
        events.append(("call", _shapes(feed)))
        return call(self, feed)

    def counting_replay(self):
        events.append(("replay", _shapes(self.static)))
        return replay(self)

    monkeypatch.setattr(graph.GraphedStep, "__init__", counting_init)
    monkeypatch.setattr(graph.GraphedStep, "__call__", counting_call)
    monkeypatch.setattr(graph.GraphedStep, "replay", counting_replay)
    forward = model.forward

    def counting_forward(feed):
        if not capturing[0]:
            events.append(("eager", _shapes(feed)))
        return forward(feed)

    model.forward = counting_forward
    return events


@pytest.mark.parametrize("route", [["--fused_step", "1"], ["--graph_step", "1"]])
def test_host_routes_leave_the_cpu_generators_where_the_reference_fit_does(route):
    """the DataLoader's base seed, the sampler's seed and one torch.rand per batch from the global torch generator, the
    negatives from NumPy's: after one epoch both generators stand where the reference loop leaves them"""
    def epoch(flags):
        model, train, runner = _setup("BPRMF", BPRMF + flags)
        loss = runner.fit(train, epoch=1)
        torch.cuda.synchronize()
        assert np.isfinite(loss)
        return model, torch.get_rng_state(), np.random.get_state()

    _, torch_ref, np_ref = epoch([])
    model, torch_st, np_st = epoch(route)
    assert ("_b2r_graphed_step" in model.__dict__) == (route[0] == "--graph_step")
    assert torch.equal(torch_st, torch_ref)
    assert len(np_st) == len(np_ref) and all(np.array_equal(x, y) for x, y in zip(np_st, np_ref))


def test_fused_step_epoch_equals_train_step_by_hand_on_the_same_batches():
    """--fused_step 1: the runner's epoch is model.train_step over the reference DataLoader's batches, each given the next
    one (already on the device) exactly when it has the same shape -- bit for bit the same losses and tables"""
    from torch.utils.data import DataLoader
    from rechorus_b200 import ops
    from rechorus_b200.runner import batch_to_device
    model, train, runner = _setup("BPRMF", BPRMF + ["--fused_step", "1"])
    steps, prefetched = [], []
    train_step = model.train_step

    def recording_step(feed, next_feed=None):
        assert next_feed is None or next_feed["item_id"].is_cuda
        prefetched.append(next_feed is not None)
        steps.append(train_step(feed, next_feed))
        return steps[-1]

    model.train_step = recording_step
    loss = runner.fit(train, epoch=1)
    # the same epoch by hand on an identically initialised model, from the same seeds
    model2, train2, _ = _setup("BPRMF", BPRMF)
    train2.actions_before_epoch()
    model2.train()
    dl = DataLoader(train2, batch_size=64, shuffle=True, num_workers=0, collate_fn=train2.collate_batch)
    batches = [batch_to_device(b, model2.device) for b in dl]
    assert len(batches) >= 3 and batches[-1]["item_id"].shape[0] < 64      # full batches and a ragged last one
    losses, want_prefetch = [], []
    ops.bprmf_step_reset()
    for k, b in enumerate(batches):
        nxt = batches[k + 1] if k + 1 < len(batches) else None
        same = nxt is not None and nxt["item_id"].shape == b["item_id"].shape
        want_prefetch.append(same)
        losses.append(model2.train_step(b, nxt if same else None))
    ops.bprmf_step_reset()
    assert prefetched == want_prefetch
    assert torch.equal(torch.stack(steps), torch.stack(losses))
    assert loss == float(np.mean(torch.stack(losses).cpu().numpy()))
    for (k, pa), (_, pb) in zip(model.named_parameters(), model2.named_parameters()):
        assert torch.equal(pa, pb), k
    ops.check_ids()


def test_host_graph_route_captures_once_and_steps_other_shapes_eagerly(monkeypatch):
    """--graph_step 1 on host SASRec batches, each padded to its own longest history: over two epochs the first full-size
    batch is captured and nothing else is; a batch of the captured shape is copied in and replayed, any other (the ragged
    last one, a full-size one of another width) runs eagerly"""
    B = 32
    model, train, runner = _setup("SASRec", SASREC + ["--graph_step", "1", "--batch_size", str(B)])
    events = _record_graph_steps(monkeypatch, model)
    losses = [runner.fit(train, epoch=e) for e in (1, 2)]
    torch.cuda.synchronize()
    n_steps = 2 * ((len(train) + B - 1) // B)
    assert all(np.isfinite(losses)) and len(events) == n_steps
    kinds = [k for k, _ in events]
    assert kinds[0] == "capture" and kinds.count("capture") == 1 and "replay" not in kinds
    captured = events[0][1]
    assert captured["item_id"][0] == B
    for kind, shapes in events[1:]:
        assert (kind == "call") == (shapes == captured), (kind, shapes, captured)
    # the case the capture policy is about: a full-size batch of another width, stepped eagerly
    assert any(k == "eager" and s["item_id"][0] == B for k, s in events) and "call" in kinds
    assert model.optimizer.t == n_steps


def test_device_graph_route_captures_again_for_another_batch_size(monkeypatch):
    """--device_batches with --graph_step 1: the full batches of an epoch share one shape, so a new batch size captures a
    new step; every later full batch is collated into the captured inputs and replayed without passing through
    GraphedStep.__call__, and the ragged last batch runs eagerly"""
    model, train, runner = _setup("NeuMF", NEUMF + ["--lr", "1e-3", "--device_batches", "77", "--graph_step", "1"])
    events = _record_graph_steps(monkeypatch, model)
    n = len(train)
    for B in (64, 48):
        del events[:]
        runner.batch_size = B
        loss = runner.fit(train, epoch=1 if B == 64 else 2)
        torch.cuda.synchronize()
        assert np.isfinite(loss) and n % B != 0
        kinds = [k for k, _ in events]
        assert kinds == ["capture"] + ["replay"] * (n // B - 1) + ["eager"], kinds
        assert all(s["item_id"][0] == B for _, s in events[:-1]) and events[-1][1]["item_id"][0] == n % B
    assert model.optimizer.t == (n + 63) // 64 + (n + 47) // 48
