"""GPU: SASRec on long histories with --tiled_attention.  The tiled attention kernels and the long last-query form against
plain float64 PyTorch (tolerances and deliberately wrong references of tests/test_gpu_seq_envelope.py), their bit identity
with the register-resident and last-query kernels wherever those accept a shape, the route ops takes with tiled=True,
b2r_seq_train_check_tiled against the launchers, and whole long-history models against the float64 oracle."""
import argparse
import types

import pytest
import torch

from oracle import rechorus_oracle as O
from tests.test_gpu_seq_envelope import (RT_CASES, TOL_GRAD, TOL_OUT, _attn64, _attn_last64, _close, _far, _runs,
                                         _spy)

pytestmark = pytest.mark.gpu


def _p(t):
    return 0 if t is None else t.data_ptr()


def _lib():
    from rechorus_b200 import lib as L
    return L.load()


def _check(rc, name):
    from rechorus_b200 import lib as L
    L.check(rc, name)


def _attention_abi(kind, q, k, v, H, live, go):
    """ctx, lse, dq, dk, dv of b2r_attention_{fwd,bwd}_<kind> (kind: rt | tiled) called through the C ABI"""
    h = _lib()
    B, L, d = q.shape
    ctx, lse = torch.empty_like(q), torch.full((B, L, H), float("nan"), device=q.device)
    dq, dk, dv = (torch.full_like(q, float("nan")) for _ in range(3))
    _check(getattr(h, f"b2r_attention_fwd_{kind}")(_p(q), _p(k), _p(v), d, _p(live), _p(ctx), _p(lse), B, L, d, H, 0),
           kind)
    args = [_p(q), _p(k), _p(v), d, _p(live), _p(ctx), _p(lse), _p(go), _p(dq), _p(dk), _p(dv), d, B, L, d, H]
    if kind == "tiled":
        ws = torch.empty(int(h.b2r_attention_bwd_tiled_workspace_bytes(B, L, H)), dtype=torch.uint8, device=q.device)
        args += [_p(ws), ws.numel()]
    _check(getattr(h, f"b2r_attention_bwd_{kind}")(*args, 0), kind)
    torch.cuda.synchronize()
    return ctx, lse, dq, dk, dv


def _inputs(B, L, d, seed, live):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, L, d, generator=g) * 2.0
    k, v, go = (torch.randn(B, L, d, generator=g) for _ in range(3))
    lv, rowmask = None, torch.ones(B, L, 1, dtype=torch.float64)
    if live:
        lv = torch.randint(1, L + 1, (B,), generator=g)
        lv[0], lv[-1] = L, 1
        rowmask = (torch.arange(L).view(1, L) < lv.view(B, 1)).unsqueeze(-1).double()
    return q, k, v, go * rowmask.float(), lv, rowmask


# --------------------------------------------------------------------------------------------------------------------
# tiled causal attention against float64
# --------------------------------------------------------------------------------------------------------------------

DK_SHAPES = {8: (64, 8), 16: (64, 4), 32: (256, 8), 64: (128, 2)}       # dk -> (d, H)


@pytest.mark.parametrize("live", [False, True])
@pytest.mark.parametrize("L", [1, 31, 33, 129, 200, 257, 511, 1024])
@pytest.mark.parametrize("dk", [8, 16, 32, 64])
def test_tiled_attention_matches_float64(dk, L, live):
    d, H = DK_SHAPES[dk]
    B = 2
    q, k, v, go, lv, rowmask = _inputs(B, L, d, 31 * L + dk + (5 if live else 0), live)
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref = _attn64(q64, k64, v64, H)
    ref.backward(go.double())
    ctx, _, dq, dk_, dv = _attention_abi("tiled", q.cuda(), k.cuda(), v.cuda(), H, None if lv is None else lv.cuda(),
                                         go.cuda())
    _close(ctx, ref * rowmask, TOL_OUT, "ctx")
    for name, a, b in (("dq", dq, q64.grad), ("dk", dk_, k64.grad), ("dv", dv, v64.grad)):
        _close(a, b, TOL_GRAD, name)
    if live:
        dead = (1 - rowmask).bool().expand(B, L, d)
        for name, t in (("ctx", ctx), ("dq", dq), ("dk", dk_), ("dv", dv)):
            assert bool((t.cpu()[dead] == 0).all()), f"dead rows of {name} are not zero"
    if L > 1:
        with torch.no_grad():
            _far(ctx, _attn64(q.double(), k.double(), v.double(), H, diag=False) * rowmask, TOL_OUT, "ctx")


def test_tiled_attention_dk64_at_d64_h1_matches_float64():
    B, L, d, H = 3, 300, 64, 1
    q, k, v, go, lv, rowmask = _inputs(B, L, d, 77, True)
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref = _attn64(q64, k64, v64, H)
    ref.backward(go.double())
    ctx, _, dq, dk, dv = _attention_abi("tiled", q.cuda(), k.cuda(), v.cuda(), H, lv.cuda(), go.cuda())
    _close(ctx, ref * rowmask, TOL_OUT, "ctx")
    for name, a, b in (("dq", dq, q64.grad), ("dk", dk, k64.grad), ("dv", dv, v64.grad)):
        _close(a, b, TOL_GRAD, name)


# --------------------------------------------------------------------------------------------------------------------
# bit identity with the register-resident and last-query kernels
# --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("live", [False, True])
@pytest.mark.parametrize("B,L,d,H", RT_CASES + [(64, 128, 64, 4), (64, 50, 64, 4), (33, 100, 32, 4)])
def test_tiled_attention_bits_equal_the_rt_kernels(B, L, d, H, live):
    q, k, v, go, lv, rowmask = _inputs(B, L, d, 13 * L + d + H, live)
    args = (q.cuda(), k.cuda(), v.cuda(), H, None if lv is None else lv.cuda(), go.cuda())
    rt = _attention_abi("rt", *args)
    tl = _attention_abi("tiled", *args)
    rows = rowmask.bool().view(B, L).cuda()
    for name, a, b in zip(("ctx", "dq", "dk", "dv"), (rt[0],) + rt[2:], (tl[0],) + tl[2:]):
        assert torch.equal(a, b), name
    assert torch.equal(rt[1][rows], tl[1][rows]), "lse"


def _last_abi(tiled, q, k, v, lengths, H, go):
    h = _lib()
    B, L, d = k.shape
    sfx = "_tiled" if tiled else ""
    ctx, prob = torch.empty(B, d, device="cuda"), torch.empty(B, H, L, device="cuda")
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(k)
    _check(getattr(h, "b2r_attention_last_fwd" + sfx)(_p(q), _p(k), _p(v), d, _p(lengths), _p(ctx), _p(prob), B, L, d, H,
                                                      0), "last_fwd")
    args = [_p(q), _p(k), _p(v), d, _p(lengths), _p(prob), _p(go), _p(dq), _p(dk), _p(dv), d, B, L, d, H]
    if tiled:
        ws = torch.empty(int(h.b2r_attention_bwd_tiled_workspace_bytes(B, L, H)), dtype=torch.uint8, device="cuda")
        args += [_p(ws), ws.numel()]
    _check(getattr(h, "b2r_attention_last_bwd" + sfx)(*args, 0), "last_bwd")
    torch.cuda.synchronize()
    return ctx, prob, dq, dk, dv


def _last_inputs(B, L, d, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, d, generator=g) * 2.0
    k, v = (torch.randn(B, L, d, generator=g) for _ in range(2))
    go = torch.randn(B, d, generator=g)
    lengths = torch.randint(1, L + 1, (B,), generator=g)
    lengths[:4] = torch.tensor([L, 1, L + 7, 0])
    return q, k, v, go, lengths


@pytest.mark.parametrize("L,d,H", [(1, 32, 4), (32, 64, 4), (33, 96, 3), (128, 128, 2), (129, 64, 8), (200, 64, 4),
                                   (255, 64, 2), (256, 64, 1), (256, 128, 16), (256, 256, 8)])
def test_long_last_query_bits_equal_the_last_query_kernels(L, d, H):
    q, k, v, go, lengths = _last_inputs(37, L, d, L + d + H)
    args = (q.cuda(), k.cuda(), v.cuda(), lengths.cuda(), H, go.cuda())
    for name, a, b in zip(("ctx", "prob", "dq", "dk", "dv"), _last_abi(False, *args), _last_abi(True, *args)):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("L,d,H", [(257, 64, 4), (300, 96, 3), (1024, 64, 1), (4096, 128, 8)])
def test_long_last_query_matches_float64(monkeypatch, L, d, H):
    from rechorus_b200 import ops
    calls = _spy(monkeypatch, "b2r_attention_last_fwd_tiled", "b2r_attention_last_bwd_tiled")
    B = 6
    q, k, v, go, lengths = _last_inputs(B, L, d, 3 * L + d + H)
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref = _attn_last64(q64, k64, v64, lengths, H)
    ref.backward(go.double())
    qc, kc, vc = (t.cuda().requires_grad_(True) for t in (q, k, v))
    out = ops.attention_last(qc, kc, vc, lengths.cuda(), H, tiled=True)
    out.backward(go.cuda())
    assert calls == [("b2r_attention_last_fwd_tiled", 0), ("b2r_attention_last_bwd_tiled", 0)], calls
    _close(out, ref, TOL_OUT, "ctx_last")
    for name, a, b in (("dq", qc.grad, q64.grad), ("dk", kc.grad, k64.grad), ("dv", vc.grad, v64.grad)):
        _close(a, b, TOL_GRAD, name)
    t = (lengths - 1).clamp(0, L - 1)
    for b in range(B):
        for name, gr in (("dk", kc.grad), ("dv", vc.grad)):
            assert bool((gr[b, int(t[b]) + 1:] == 0).all()), f"{name} rows beyond t* of sequence {b} are not zero"
    with torch.no_grad():
        _far(out, _attn_last64(q.double(), k.double(), v.double(), lengths, H, shift=2), TOL_OUT, "ctx_last")


# --------------------------------------------------------------------------------------------------------------------
# the route ops takes with tiled=True
# --------------------------------------------------------------------------------------------------------------------

FULL_ROUTES = [((50, 64, 4), "rt"), ((128, 32, 1), "rt"), ((86, 128, 4), "rt"), ((128, 64, 1), "live"),
               ((84, 128, 2), "live"), ((50, 96, 2), "live"), ((87, 128, 4), "tiled"), ((129, 64, 4), "tiled"),
               ((129, 64, 1), "tiled"), ((85, 128, 2), "tiled"), ((300, 256, 8), "tiled")]


@pytest.mark.parametrize("shape,route", FULL_ROUTES)
def test_tiled_keyword_keeps_todays_kernels_inside_the_old_envelope(monkeypatch, shape, route):
    from rechorus_b200 import ops
    L, d, H = shape
    names = [f"b2r_attention_{dr}_{r}" for r in ("rt", "live", "tiled") for dr in ("fwd", "bwd")]
    calls = _spy(monkeypatch, *names)
    q, k, v = (torch.randn(2, L, d, device="cuda", requires_grad=True) for _ in range(3))
    ops.causal_attention(q, k, v, H, live=torch.tensor([L, 1], device="cuda"), tiled=True).sum().backward()
    torch.cuda.synchronize()
    assert calls == [(f"b2r_attention_fwd_{route}", 0), (f"b2r_attention_bwd_{route}", 0)], calls


@pytest.mark.parametrize("L,route", [(1, ""), (256, ""), (257, "_tiled"), (600, "_tiled")])
def test_tiled_keyword_keeps_the_last_query_kernels_up_to_256(monkeypatch, L, route):
    from rechorus_b200 import ops
    calls = _spy(monkeypatch, "b2r_attention_last_fwd", "b2r_attention_last_bwd", "b2r_attention_last_fwd_tiled",
                 "b2r_attention_last_bwd_tiled")
    d, H = 64, 4
    ql = torch.randn(2, d, device="cuda", requires_grad=True)
    k, v = (torch.randn(2, L, d, device="cuda", requires_grad=True) for _ in range(2))
    ops.attention_last(ql, k, v, torch.tensor([L, 1], device="cuda"), H, tiled=True).sum().backward()
    torch.cuda.synchronize()
    assert calls == [(f"b2r_attention_last_fwd{route}", 0), (f"b2r_attention_last_bwd{route}", 0)], calls


AGREE_DH = [(32, 4), (64, 4), (64, 1), (96, 3), (128, 4), (128, 2), (128, 1), (256, 8), (256, 4), (288, 4)]
AGREE_L = [1, 85, 87, 128, 129, 256, 257, 600]


@pytest.mark.parametrize("d,H", AGREE_DH)
def test_seq_train_check_tiled_agrees_with_the_launchers(d, H):
    from rechorus_b200 import lib as Lb
    from rechorus_b200 import ops
    h = Lb.load()
    B = 2
    gam, bet = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
    for L in AGREE_L:
        lengths = torch.tensor([L, 1], device="cuda")
        q, k, v = (torch.randn(B, L, d, device="cuda", requires_grad=True) for _ in range(3))
        ql = torch.randn(B, d, device="cuda", requires_grad=True)

        def full_block():
            ctx = ops.causal_attention(q, k, v, H, live=lengths, tiled=True)
            ops.add_layernorm(ctx, ctx.detach(), gam, bet).sum().backward()

        def last_block():
            ctx = ops.attention_last(ql, k, v, lengths, H, tiled=True)
            ops.add_layernorm(ctx, ctx.detach(), gam, bet).sum().backward()

        for verdict_args, fn in (((L, d, H, 1, 0), full_block), ((L, d, H, 0, Lb.SEQ_LAST_QUERY), last_block)):
            accepted = h.b2r_seq_train_check_tiled(*verdict_args) == 0
            assert _runs(fn) == accepted, (verdict_args, h.b2r_last_error().decode())


# --------------------------------------------------------------------------------------------------------------------
# whole models
# --------------------------------------------------------------------------------------------------------------------

def _model(d, H, layers, hm, dropout=0.0, scale=10.0, seed=None, n_items=300):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    p = plugin.SASRec.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(["--emb_size", str(d), "--num_heads", str(H), "--num_layers", str(layers), "--history_max", str(hm),
                      "--num_neg", "4", "--tiled_attention", "1", "--dropout", str(dropout)])
    a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_unused.pt"
    torch.manual_seed(d + hm if seed is None else seed)
    m = plugin.SASRec(a, types.SimpleNamespace(n_users=10, n_items=n_items)).to(a.device)
    with torch.no_grad():
        for name, q in m.named_parameters():
            if "layer_norm" not in name:
                q.mul_(scale)                                  # trained-scale weights: softmaxes far from uniform
    return m


def _batch(hm, B=12, C=5, n_items=300, seed=0):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, hm + 1, (B,), generator=g)
    lengths[0], lengths[1] = hm, 1
    hist = torch.randint(1, n_items, (B, hm), generator=g) * (torch.arange(hm).view(1, hm) < lengths.view(B, 1))
    iid = torch.randint(1, n_items, (B, C), generator=g)
    batch = {"history_items": hist, "lengths": lengths, "item_id": iid}
    feed = {k: v.cuda() for k, v in batch.items()}
    feed.update(user_id=torch.zeros(B, dtype=torch.int64, device="cuda"), batch_size=B, phase="train")
    return batch, feed


def _step(m, feed):
    from rechorus_b200 import ops
    m.zero_grad()
    out = m(feed)
    loss = m.loss(out)
    loss.backward()
    ops.check_ids()
    return out["prediction"].detach(), loss.detach(), {k: q.grad.detach().clone() for k, q in m.named_parameters()}


LONG_GRID = [(64, 4, 2, 200), (64, 1, 2, 200), (64, 4, 1, 512), (128, 4, 2, 150), (256, 8, 2, 100), (64, 2, 3, 300)]


@pytest.mark.parametrize("lastq", [True, False])
@pytest.mark.parametrize("d,H,layers,hm", LONG_GRID)
def test_long_history_sasrec_matches_float64_oracle(monkeypatch, d, H, layers, hm, lastq):
    from rechorus_b200 import plugin
    monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
    m = _model(d, H, layers, hm)
    batch, feed = _batch(hm, seed=d * 1000 + hm)
    w64 = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    pred64, loss64, g64 = O.loss_and_grads("SASRec", w64, batch, H)
    m.train()
    pred, loss, grads = _step(m, feed)
    _close(pred, pred64, TOL_OUT, "prediction")
    _close(loss.view(1), loss64.view(1), TOL_OUT, "loss")
    assert sorted(grads) == sorted(g64)
    for k, g in grads.items():
        _close(g, g64[k], TOL_GRAD, k)
    m.eval()
    with torch.no_grad():
        _close(m(feed)["prediction"], pred64, TOL_OUT, "eval prediction")


def test_last_query_block_equals_full_block_with_dropout_at_200(monkeypatch):
    from rechorus_b200 import plugin
    res = {}
    for lastq in (True, False):
        monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
        m = _model(64, 4, 2, 200, dropout=0.2, scale=3.0, seed=5)
        m.set_dropout_rng_state(11, 4)
        m.train()
        res[lastq] = _step(m, _batch(200, seed=9)[1])
    (pa, la, ga), (pb, lb, gb) = res[True], res[False]
    _close(pa, pb, 1e-5, "prediction")
    _close(la.view(1), lb.view(1), 1e-5, "loss")
    for k in ga:
        _close(ga[k], gb[k], 2e-5, k)


def test_two_runs_give_identical_bits():
    runs = []
    for _ in range(2):
        m = _model(64, 4, 2, 300, dropout=0.2, seed=2)
        m.set_dropout_rng_state(7, 1)
        m.train()
        runs.append(_step(m, _batch(300, B=64, seed=4)[1]))
    (pa, la, ga), (pb, lb, gb) = runs
    assert torch.equal(pa, pb) and torch.equal(la, lb)
    for k in ga:
        assert torch.equal(ga[k], gb[k]), k


def test_graphed_steps_equal_eager_steps_at_history_200():
    from rechorus_b200 import ops
    from rechorus_b200.graph import GraphedStep
    from rechorus_b200.optim import RowSparseOptimizer

    def build(device_clock):
        m = _model(64, 4, 2, 200, scale=3.0, seed=3)
        m.set_table_mode("fused")
        m.optimizer = RowSparseOptimizer(m, "Adam", lr=1e-2, l2=1e-5, eps=1e-3, device_clock=device_clock)
        m.train()
        return m

    feeds = [_batch(200, B=64, C=6, seed=s)[1] for s in range(7)]
    eager, graphed = build(False), build(True)
    step = GraphedStep(graphed, feeds[0], warmup=2)
    losses_e = []
    for f in [feeds[0], feeds[0]] + feeds[1:]:
        eager.optimizer.zero_grad()
        ls = eager.loss(eager(f))
        ls.backward()
        eager.optimizer.step()
        losses_e.append(float(ls.detach()))
    losses_g = [float(step(f)) for f in feeds[1:]]
    torch.cuda.synchronize()
    assert graphed.optimizer.sync_clock() == eager.optimizer.t == 8
    tol_l = 1e-6 * max(1.0, max(losses_e))
    for a, b in zip(losses_g, losses_e[2:]):
        assert abs(a - b) <= tol_l, (losses_g, losses_e)
    for (k, pa), (_, pb) in zip(graphed.named_parameters(), eager.named_parameters()):
        assert (pa - pb).abs().max() <= 1e-6, k
    ops.check_ids()


# --------------------------------------------------------------------------------------------------------------------
# parity with the reference (tests/golden/make_long_history_golden.py): history_max 200, 2 blocks, p = 0.2 and p = 0
# --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("lastq", [True, False])
@pytest.mark.parametrize("p0", [False, True])
def test_sasrec_long_fixture_parity(monkeypatch, lastq, p0):
    from rechorus_b200 import plugin
    from tests.test_gpu_dropout import _feed, _load
    monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
    meta, z, w, batch, g_ref = _load("sasrec_long")
    m = _model(meta["d"], meta["num_heads"], meta["num_layers"], meta["history_max"], dropout=0.0 if p0 else meta["p"],
               n_items=meta["n_items"])
    m.load_state_dict(w)
    m.set_dropout_rng_state(meta["seed"], meta["step"])
    m.train()
    pred, loss, grads = _step(m, _feed(batch, meta["B"]))
    pre = "p0:" if p0 else ""
    ref_pred, ref_loss = torch.from_numpy(z[pre + "prediction"]), torch.from_numpy(z[pre + "loss"])
    assert (pred.cpu() - ref_pred).abs().max() <= 1e-5
    assert abs(float(loss) - float(ref_loss)) <= 1e-5
    for k, g in grads.items():
        ref = torch.from_numpy(z[pre + "g:" + k])
        assert (g.cpu() - ref).abs().max() <= 1e-5, (k, float((g.cpu() - ref).abs().max()))
    if not p0:                                                  # the masks matter: p = 0 results are far from these
        assert (pred.cpu() - torch.from_numpy(z["p0:prediction"])).abs().max() > 1e-3
