"""GPU: dropout fused into the Linear and residual-LayerNorm kernels (b2r_dropout, include/b200rec.h).  The kernels' mask
bits against tests/dropout_oracle.dropout_mask, NeuMF / SASRec with --dropout 0.2 against fixtures the reference's own
code produced with those masks (tests/golden/make_dropout_golden.py), the last-query block against the full block, eval
mode, CUDA-graph replay, the runner's graphed route and the overlay."""
import argparse
import ast
import os
import types

import numpy as np
import pytest
import torch

from oracle import rechorus_oracle as O
from tests import dropout_oracle as D

pytestmark = pytest.mark.gpu
TOL = 1e-5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SEED = 0x0123456789ABCDEF


def _drop(p, site, step=3):
    from rechorus_b200 import ops
    st = ops.DropoutState(SEED, torch.device("cuda", 0))
    st.set(SEED, step)
    return ops.Drop(st.tick(), p, site)


# ------------------------------------------------------------------------------------------------------
# 1-2: mask bits
# ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("p", [0.1, 0.5, 1.0])
@pytest.mark.parametrize("M,N,K,tc", [(4608, 64, 64, True), (4100, 16, 128, True), (300, 13, 24, False),
                                      (77, 64, 64, False)])
def test_linear_dropout_forward_returns_mask_times_scale(p, M, N, K, tc):
    from rechorus_b200 import ops
    drop = _drop(p, site=2)
    x = torch.zeros(M, K, device="cuda")
    W = torch.zeros(N, K, device="cuda")
    b = torch.ones(N, device="cuda")
    y = ops.linear_fwd_dropout(x, W, b, True, drop, tc)
    m = D.dropout_mask(SEED, 3, 2, np.arange(M), np.zeros(M), N, p)
    assert torch.equal(y.cpu(), torch.from_numpy(m).float() * D.dropout_scale(p))


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_tensor_core_epilogue_is_the_plain_output_times_mask(p):
    from rechorus_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    M, N, K = 8192, 64, 128
    x = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) * 0.1
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    y0 = ops.linear_fwd_tc(x, W, b, True)
    y = ops.linear_fwd_dropout(x, W, b, True, _drop(p, site=0), True)
    m = torch.from_numpy(D.dropout_mask(SEED, 3, 0, np.arange(M), np.zeros(M), N, p)).cuda().bool()
    s = D.dropout_scale(p)
    assert torch.equal(y, torch.where(m, y0 * s, torch.zeros_like(y0)))


def _ln_case(d, mapping, p, B=37, L=11):
    """forward and backward of add_layernorm with dropout; returns (x, res, y, dx, dres, mask)"""
    from rechorus_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(d)
    lengths = torch.randint(1, L + 3, (B,), device="cuda", generator=g)       # some beyond L: clamped as select_last does
    shape = (B, L, d) if mapping == "full" else (B, d)
    x = torch.randn(*shape, device="cuda", generator=g).requires_grad_(True)
    res = torch.randn(*shape, device="cuda", generator=g).requires_grad_(True)
    gamma = (1 + 0.1 * torch.randn(d, device="cuda", generator=g)).requires_grad_(True)
    beta = (0.1 * torch.randn(d, device="cuda", generator=g)).requires_grad_(True)
    drop = _drop(p, site=5)
    if mapping == "full":
        y = ops.add_layernorm(x, res, gamma, beta, drop=drop)
        bb, tt = np.meshgrid(np.arange(B), np.arange(L), indexing="ij")
        mask = D.dropout_mask(SEED, 3, 5, bb.reshape(-1), tt.reshape(-1), d, p).reshape(B, L, d)
    else:
        y = ops.add_layernorm(x, res, gamma, beta, drop=drop, lengths=lengths, seq_len=L)
        t = (lengths.cpu() - 1).clamp(0, L - 1).numpy()
        mask = D.dropout_mask(SEED, 3, 5, np.arange(B), t, d, p)
    dy = torch.randn_like(y)
    y.backward(dy)
    return x, res, gamma, beta, y, x.grad, res.grad, torch.from_numpy(mask).cuda().bool()


@pytest.mark.parametrize("p", [0.1, 0.5, 1.0])
@pytest.mark.parametrize("d", [64, 32, 30, 20, 200])
@pytest.mark.parametrize("mapping", ["full", "last"])
def test_layernorm_dropout_mask_bits(p, d, mapping):
    """backward: dx = dres * mask * s bit for bit; forward: identical to the plain kernel on torch.where(mask, x * s, 0)"""
    from rechorus_b200 import ops
    x, res, gamma, beta, y, dx, dres, mask = _ln_case(d, mapping, p)
    s = D.dropout_scale(p)
    assert torch.equal(dx, torch.where(mask, dres * s, torch.zeros_like(dres)))
    with torch.no_grad():
        y0 = ops.add_layernorm(torch.where(mask, x * s, torch.zeros_like(x)), res, gamma, beta)
    assert torch.equal(y.detach(), y0)


# ------------------------------------------------------------------------------------------------------
# 3-6: fixture parity, last-query block, padding, eval mode
# ------------------------------------------------------------------------------------------------------

def _load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = ast.literal_eval(str(z["meta"]))
    pick = lambda pre: {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre)}  # noqa: E731
    return meta, z, pick("w:"), pick("in:"), pick("g:")


def _build(model_name, meta, weights, mode="dense", p=None):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, model_name)
    ap = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    extra = ["--emb_size", str(meta["d"]), "--table_mode", mode, "--dropout", str(meta["p"] if p is None else p)]
    if model_name == "NeuMF":
        extra += ["--layers", str(meta["layers"])]
    else:
        extra += ["--history_max", str(meta["history_max"]), "--num_layers", str(meta["num_layers"]),
                  "--num_heads", str(meta["num_heads"])]
    a = ap.parse_args(extra)
    a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_unused.pt"
    m = cls(a, types.SimpleNamespace(n_users=meta.get("n_users", 10), n_items=meta["n_items"])).to(a.device)
    m.load_state_dict(weights)
    m.set_table_mode(mode)
    m.set_dropout_rng_state(meta["seed"], meta["step"])
    m.train()
    return m


def _feed(batch, B):
    out = {k: v.cuda() for k, v in batch.items()}
    out["batch_size"], out["phase"] = B, "train"
    return out


def _step(m, feed, mode="dense"):
    from rechorus_b200 import ops
    if mode == "fused":
        from rechorus_b200.optim import RowSparseOptimizer
        m.optimizer = RowSparseOptimizer(m, "SGD", lr=0.0)
        m.optimizer.zero_grad()
    out = m(feed)
    loss = m.loss(out)
    loss.backward()
    ops.check_ids()
    grads = {}
    for k, q in m.named_parameters():
        if mode == "fused" and ops.table_mode(q) == "fused":
            continue
        g = q.grad
        grads[k] = (g.to_dense() if g.is_sparse else g).cpu() if g is not None else None
    return out["prediction"].detach().cpu(), float(loss), grads


@pytest.mark.parametrize("mode", ["dense", "sparse", "fused"])
@pytest.mark.parametrize("model_name,fixture", [("NeuMF", "neumf_dropout"), ("SASRec", "sasrec_dropout")])
def test_fixture_parity(model_name, fixture, mode):
    meta, z, w, batch, g_ref = _load(fixture)
    m = _build(model_name, meta, w, mode)
    pred, loss, grads = _step(m, _feed(batch, meta["B"]), mode)
    pred_ref = torch.from_numpy(z["prediction"])
    assert (pred - pred_ref).abs().max() <= TOL
    assert abs(loss - float(z["loss"])) <= TOL
    assert np.array_equal(O.gt_rank(pred.numpy()), O.gt_rank(pred_ref.numpy()))
    assert m.dropout_rng_state() == (meta["seed"], meta["step"] + 1)
    for k, g in grads.items():
        g = torch.zeros_like(g_ref[k]) if g is None else g
        assert (g - g_ref[k]).abs().max() <= TOL, (k, float((g - g_ref[k]).abs().max()))


def test_sasrec_last_query_block_equals_full_block(monkeypatch):
    from rechorus_b200 import plugin
    meta, z, w, batch, _ = _load("sasrec_dropout")
    feed = _feed(batch, meta["B"])
    res = {}
    for lastq in (True, False):
        monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
        res[lastq] = _step(_build("SASRec", meta, w), feed)
    (pa, la, ga), (pb, lb, gb) = res[True], res[False]
    assert (pa - pb).abs().max() <= 1e-6 and abs(la - lb) <= 1e-6
    for k in ga:
        assert (ga[k] - gb[k]).abs().max() <= 1e-6, k


def test_sasrec_extra_right_padding_changes_nothing():
    meta, z, w, batch, _ = _load("sasrec_dropout")
    pred, loss, grads = _step(_build("SASRec", meta, w), _feed(batch, meta["B"]))
    padded = dict(batch)
    padded["history_items"] = torch.from_numpy(z["pad:in:history_items"])
    padded["history_times"] = torch.zeros_like(padded["history_items"])
    pred_p, loss_p, grads_p = _step(_build("SASRec", meta, w), _feed(padded, meta["B"]))
    assert (pred - pred_p).abs().max() <= 1e-6 and abs(loss - loss_p) <= 1e-6
    assert (pred_p - torch.from_numpy(z["pad:prediction"])).abs().max() <= TOL
    for k in grads:
        assert (grads[k] - grads_p[k]).abs().max() <= 1e-6, k


@pytest.mark.parametrize("model_name,fixture", [("NeuMF", "neumf_dropout"), ("SASRec", "sasrec_dropout")])
def test_eval_mode_equals_no_dropout(model_name, fixture):
    meta, z, w, batch, _ = _load(fixture)
    feed = _feed(batch, meta["B"])
    m, m0 = _build(model_name, meta, w), _build(model_name, meta, w, p=0.0)
    m.eval()
    m0.eval()
    with torch.no_grad():
        assert torch.equal(m(feed)["prediction"], m0(feed)["prediction"])
    assert m.dropout_rng_state() == (meta["seed"], meta["step"])            # evaluation does not tick


# ------------------------------------------------------------------------------------------------------
# 7-9: CUDA graph, runner, overlay
# ------------------------------------------------------------------------------------------------------

def _graph_model(name, flags, device_clock):
    from rechorus_b200 import plugin
    from rechorus_b200.optim import RowSparseOptimizer
    cls = getattr(plugin, name)
    a = cls.parse_model_args(argparse.ArgumentParser()).parse_args(flags + ["--table_mode", "fused", "--dropout", "0.2"])
    a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_graph.pt"
    torch.manual_seed(3)
    m = cls(a, types.SimpleNamespace(n_users=200, n_items=300)).to(a.device)
    with torch.no_grad():
        for q in m.parameters():
            q.mul_(10.0)
    m.optimizer = RowSparseOptimizer(m, "Adam", lr=1e-2, l2=1e-5, eps=1e-3, device_clock=device_clock)
    m.train()
    return m


def _graph_feeds(name, n, B=64, C=6, L=9):
    g = torch.Generator().manual_seed(8)
    out = []
    for _ in range(n):
        f = {"user_id": torch.randint(1, 200, (B,), generator=g).cuda(),
             "item_id": torch.randint(1, 300, (B, C), generator=g).cuda(), "batch_size": B, "phase": "train"}
        if name == "SASRec":
            lengths = torch.randint(1, L + 1, (B,), generator=g)
            lengths[0] = L
            f["history_items"] = (torch.randint(1, 300, (B, L), generator=g)
                                  * (torch.arange(L).view(1, L) < lengths.view(B, 1))).cuda()
            f["lengths"] = lengths.cuda()
        out.append(f)
    return out


@pytest.mark.parametrize("name,flags", [("NeuMF", ["--emb_size", "32", "--layers", "[32, 16]"]),
                                        ("SASRec", ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2",
                                                    "--history_max", "9"])])
def test_graphed_dropout_steps_equal_eager_steps(name, flags):
    from rechorus_b200.graph import GraphedStep
    feeds = _graph_feeds(name, 7)
    eager = _graph_model(name, flags, device_clock=False)
    graphed = _graph_model(name, flags, device_clock=True)
    step = GraphedStep(graphed, feeds[0], warmup=2)
    losses_e = []
    for f in [feeds[0], feeds[0]] + feeds[1:]:
        eager.optimizer.zero_grad()
        ls = eager.loss(eager(f))
        ls.backward()
        eager.optimizer.step()
        losses_e.append(float(ls))
    losses_g = [float(step(f)) for f in feeds[1:]]
    torch.cuda.synchronize()
    assert graphed.optimizer.sync_clock() == eager.optimizer.t == 8
    assert graphed.dropout_rng_state()[1] == eager.dropout_rng_state()[1] == 8
    tol_l = 1e-6 * max(1.0, max(losses_e))
    for a, b in zip(losses_g, losses_e[2:]):
        assert abs(a - b) <= tol_l, (losses_g, losses_e)
    for (k, pa), (_, pb) in zip(graphed.named_parameters(), eager.named_parameters()):
        assert (pa - pb).abs().max() <= 1e-6, k


def test_runner_graph_step_with_dropout_takes_the_graphed_route():
    import sys
    sys.path.insert(0, GOLDEN)
    import fit_corpus
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner

    def run():
        ap = plugin.NeuMF.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
        a = ap.parse_args(["--emb_size", "32", "--layers", "[32]", "--num_neg", "5", "--batch_size", "64", "--num_workers",
                           "0", "--lr", "0.001", "--optimizer", "Adam", "--table_mode", "fused", "--fused_optimizer", "1",
                           "--graph_step", "1", "--dropout", "0.2"])
        a.device, a.model_path, a.log_file = torch.device("cuda", 0), "/tmp/_b2r_gsd.pt", ""
        corpus = fit_corpus.build()
        torch.manual_seed(1)
        np.random.seed(1)
        model = plugin.NeuMF(a, corpus).to(a.device)
        train = plugin.NeuMF.Dataset(model, corpus, "train")
        runner = BaseRunner(a)
        ls = [runner.fit(train, epoch=e) for e in (1, 2)]
        torch.cuda.synchronize()
        return model, ls

    m1, l1 = run()
    m2, l2 = run()
    assert "_b2r_graphed_step" in m1.__dict__ and all(np.isfinite(l1))
    assert l1 == l2
    for (k, pa), (_, pb) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(pa, pb), k


@pytest.mark.skipif(not os.path.isfile(os.path.join(os.path.dirname(GOLDEN), "..", "oracle", "_ref", "src", "main.py")),
                    reason="no unmodified reference staged in oracle/_ref")
def test_overlay_neumf_with_dropout_trains(tmp_path):
    from tests import test_gpu_overlay as OV
    tmp = str(tmp_path)
    OV._dataset(tmp)
    losses, metrics, ckpt, out = OV._run(tmp, "neumf_drop", OV.OVERLAY, "NeuMF",
                                         ["--num_neg", "2", "--layers", "[32, 16]", "--dropout", "0.2", "--epoch", "1"], "0")
    assert losses and all(np.isfinite(losses)), out[-2000:]
