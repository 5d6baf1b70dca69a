"""GPU: SASRec's kernels against plain float64 PyTorch on the CPU (same fp32 inputs) at the edges of their shape envelope:
causal attention on both routes, the last-query attention, the history embedding with its position-table gradient, the
residual LayerNorm, and whole SASRec models against the float64 oracle.  A result passes when max |err| <= 1e-5 *
max(1, max |ref|) (outputs) or 2e-5 * max(1, max |ref|) (gradients).  Every kernel group must also FAIL against a
deliberately wrong float64 reference, so a loose tolerance or a reference that echoes the kernel cannot pass unnoticed.
Last, b2r_seq_train_check's verdict is compared with what the launchers do."""
import argparse
import math
import types

import pytest
import torch

from oracle import rechorus_oracle as O

pytestmark = pytest.mark.gpu
TOL_OUT, TOL_GRAD = 1e-5, 2e-5


def _err(got, ref):
    got, ref = got.detach().cpu().double(), ref.detach().cpu().double()
    return float((got - ref).abs().max()), max(1.0, float(ref.abs().max()))


def _close(got, ref, tol, what):
    e, s = _err(got, ref)
    assert e <= tol * s, f"{what}: max |err| {e:.3e} > {tol:g} * {s:.4g}"


def _far(got, ref, tol, what):
    e, s = _err(got, ref)
    assert e > tol * s, f"{what}: the kernel also matches the deliberately wrong reference ({e:.3e})"


def _spy(monkeypatch, *names):
    """record (entry point, return code) of the library calls ops makes"""
    from rechorus_b200 import lib as L
    h, calls = L.load(), []
    for n in names:
        def wrap(*a, _fn=getattr(h, n), _n=n):
            rc = _fn(*a)
            calls.append((_n, rc))
            return rc
        monkeypatch.setattr(h, n, wrap)
    return calls


# --------------------------------------------------------------------------------------------------------------------
# causal attention
# --------------------------------------------------------------------------------------------------------------------

def _attn64(q, k, v, H, diag=True):
    """layers.py:52-63 in float64.  diag=False is the wrong reference: a query does not see its own key (row 0 then sees
    nothing and is set to 0, as layers.py:61 does with NaN)."""
    B, L, d = q.shape
    dk = d // H

    def split(t):
        return t.view(B, L, H, dk).transpose(1, 2)

    s = split(q) @ split(k).transpose(-1, -2) / math.sqrt(dk)
    keep = torch.ones(L, L, dtype=torch.bool).tril(0 if diag else -1)
    p = torch.nan_to_num(torch.softmax(s.masked_fill(~keep, float("-inf")), dim=-1), nan=0.0)
    return (p @ split(v)).transpose(1, 2).reshape(B, L, d)


# (B, L, d, H) the register-resident route takes (d / H in {8, 16, 32}); the last rows sit exactly at the largest L its
# backward accepts for that (d, H): (5 L (d + 4) + 2 L H) * 4 B <= 227 KB
RT_CASES = [(3, 1, 32, 4), (3, 31, 64, 4), (3, 32, 96, 3), (3, 33, 64, 8), (2, 63, 32, 2), (2, 65, 128, 8),
            (2, 127, 64, 2), (2, 128, 64, 4), (2, 128, 32, 1), (2, 128, 64, 8),
            (2, 86, 128, 4), (2, 85, 128, 8), (2, 83, 128, 16), (2, 114, 96, 3), (2, 113, 96, 6), (2, 44, 256, 8),
            (2, 42, 256, 32)]
# (B, L, d, H) on the shared-memory kernels, the only route for d / H outside {8, 16, 32}.  (2, 84, 128, 2) and
# (2, 47, 256, 4) are the largest L their backward accepts: (4 L (d + 1) + H L (L + 1)) * 4 B <= 227 KB
V1_CASES = [(3, 1, 64, 1), (3, 33, 128, 2), (2, 63, 64, 1), (2, 128, 64, 1), (2, 31, 256, 4), (2, 84, 128, 2),
            (2, 47, 256, 4),
            (3, 17, 16, 4), (2, 100, 16, 4), (3, 7, 12, 1), (3, 40, 48, 4), (2, 128, 48, 1), (2, 64, 96, 4),
            (2, 50, 96, 2), (2, 60, 128, 1), (2, 40, 256, 2)]

def _check_attention(monkeypatch, B, L, d, H, live, route):
    from rechorus_b200 import ops
    calls = _spy(monkeypatch, "b2r_attention_fwd_rt", "b2r_attention_bwd_rt", "b2r_attention_fwd_live",
                 "b2r_attention_bwd_live")
    g = torch.Generator().manual_seed(1000 * L + 10 * d + H + (7 if live else 0))
    q = torch.randn(B, L, d, generator=g) * 2.0                # scores ~ N(0, 4): softmax rows far from uniform
    k, v, go = (torch.randn(B, L, d, generator=g) for _ in range(3))
    lv, rowmask = None, torch.ones(B, L, 1, dtype=torch.float64)
    if live:
        lv = torch.randint(1, L + 1, (B,), generator=g)
        lv[0], lv[-1] = L, 1
        rowmask = (torch.arange(L).view(1, L) < lv.view(B, 1)).unsqueeze(-1).double()
    go = go * rowmask.float()                                  # dead rows receive no upstream gradient
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref = _attn64(q64, k64, v64, H)
    ref.backward(go.double())
    qc, kc, vc = (t.cuda().requires_grad_(True) for t in (q, k, v))
    out = ops.causal_attention(qc, kc, vc, H, live=None if lv is None else lv.cuda())
    out.backward(go.cuda())
    torch.cuda.synchronize()
    ran = sorted({n for n, _ in calls})
    if route == "rt":
        assert ran == ["b2r_attention_bwd_rt", "b2r_attention_fwd_rt"] and all(rc == 0 for _, rc in calls), calls
    else:
        assert ran == ["b2r_attention_bwd_live", "b2r_attention_fwd_live"] and all(rc == 0 for _, rc in calls), calls
    _close(out, ref * rowmask, TOL_OUT, "ctx")
    for name, a, b in (("dq", qc.grad, q64.grad), ("dk", kc.grad, k64.grad), ("dv", vc.grad, v64.grad)):
        _close(a, b, TOL_GRAD, name)
    if live:
        dead = (1 - rowmask).bool().expand(B, L, d)
        for name, t in (("ctx", out), ("dq", qc.grad), ("dk", kc.grad), ("dv", vc.grad)):
            assert bool((t.detach().cpu()[dead] == 0).all()), f"dead rows of {name} are not zero"
    with torch.no_grad():
        _far(out, _attn64(q.double(), k.double(), v.double(), H, diag=False) * rowmask, TOL_OUT, "ctx")


@pytest.mark.parametrize("live", [False, True])
@pytest.mark.parametrize("B,L,d,H", RT_CASES)
def test_causal_attention_rt_route_matches_float64(monkeypatch, B, L, d, H, live):
    _check_attention(monkeypatch, B, L, d, H, live, "rt")


@pytest.mark.parametrize("live", [False, True])
@pytest.mark.parametrize("B,L,d,H", V1_CASES)
def test_causal_attention_shared_memory_route_matches_float64(monkeypatch, B, L, d, H, live):
    _check_attention(monkeypatch, B, L, d, H, live, "v1")


# --------------------------------------------------------------------------------------------------------------------
# last-query attention
# --------------------------------------------------------------------------------------------------------------------

def _attn_last64(q, k, v, lengths, H, shift=1):
    """row t* = clamp(len - shift, 0, L - 1) of the causal attention, float64; shift=1 is select_last's row (SASRec.py:76),
    shift=2 the wrong reference"""
    B, L, d = k.shape
    dk = d // H
    t = (lengths - shift).clamp(0, L - 1)
    rows = []
    for b in range(B):
        n = int(t[b]) + 1
        kh, vh = (x[b, :n].view(n, H, dk).transpose(0, 1) for x in (k, v))       # [H, n, dk]
        p = torch.softmax(q[b].view(H, 1, dk) @ kh.transpose(-1, -2) / math.sqrt(dk), dim=-1)
        rows.append((p @ vh).reshape(d))
    return torch.stack(rows)


LAST_CASES = [(1, 32, 4), (32, 64, 4), (33, 96, 3), (128, 128, 2), (129, 64, 8), (255, 64, 2), (256, 64, 1),
              (256, 128, 16), (256, 256, 8)]


@pytest.mark.parametrize("L,d,H", LAST_CASES)
def test_attention_last_matches_float64(L, d, H):
    from rechorus_b200 import ops
    B = 6
    g = torch.Generator().manual_seed(L * 10 + d + H)
    q = torch.randn(B, d, generator=g) * 2.0
    k, v = (torch.randn(B, L, d, generator=g) for _ in range(2))
    go = torch.randn(B, d, generator=g)
    lengths = torch.randint(1, L + 1, (B,), generator=g)
    lengths[:4] = torch.tensor([L, 1, L + 7, 0])                # full, shortest, and two clamped like select_last
    q64, k64, v64 = (t.double().requires_grad_(True) for t in (q, k, v))
    ref = _attn_last64(q64, k64, v64, lengths, H)
    ref.backward(go.double())
    qc, kc, vc = (t.cuda().requires_grad_(True) for t in (q, k, v))
    out = ops.attention_last(qc, kc, vc, lengths.cuda(), H)
    out.backward(go.cuda())
    _close(out, ref, TOL_OUT, "ctx_last")
    for name, a, b in (("dq", qc.grad, q64.grad), ("dk", kc.grad, k64.grad), ("dv", vc.grad, v64.grad)):
        _close(a, b, TOL_GRAD, name)
    t = (lengths - 1).clamp(0, L - 1)
    for b in range(B):
        for name, gr in (("dk", kc.grad), ("dv", vc.grad)):
            assert bool((gr[b, int(t[b]) + 1:] == 0).all()), f"{name} rows beyond t* of sequence {b} are not zero"
    if L > 1:
        with torch.no_grad():
            _far(out, _attn_last64(q.double(), k.double(), v.double(), lengths, H, shift=2), TOL_OUT, "ctx_last")


# --------------------------------------------------------------------------------------------------------------------
# history embedding and the position-table gradient
# --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("p_rows", [200, 201, 257])
def test_embed_history_position_table_gradient_matches_float64(monkeypatch, p_rows, d):
    """200 rows: the shared-memory small-table kernel (G = 256 / d copies fill exactly 200 KB); 201 and 257 rows: it
    returns B2R_E_UNSUPPORTED and the plan route computes the gradient"""
    from rechorus_b200 import ops
    calls = _spy(monkeypatch, "b2r_small_table_grad")
    g = torch.Generator().manual_seed(p_rows + d)
    n_items, L, B = 50, p_rows - 1, 16
    I, P = torch.randn(n_items, d, generator=g), torch.randn(p_rows, d, generator=g)
    lengths = torch.randint(1, L + 1, (B,), generator=g)
    lengths[0], lengths[1] = L, 1
    hist = torch.randint(1, n_items, (B, L), generator=g) * (torch.arange(L).view(1, L) < lengths.view(B, 1))
    valid = (hist > 0).long()
    pos = (lengths.view(B, 1) - torch.arange(L).view(1, L)) * valid
    gx = torch.randn(B, L, d, generator=g) * valid.unsqueeze(-1)      # padded positions carry zero gradient
    I64, P64 = I.double().requires_grad_(True), P.double().requires_grad_(True)
    x64 = I64[hist] + P64[pos]
    x64.backward(gx.double())
    Ic, Pc = I.cuda().requires_grad_(True), P.cuda().requires_grad_(True)
    x = ops.embed_history(Ic, Pc, hist.cuda(), lengths.cuda())
    x.backward(gx.cuda())
    ops.check_ids()
    assert calls == [("b2r_small_table_grad", 0 if p_rows == 200 else -3)], calls
    _close(x, x64, TOL_OUT, "x")
    _close(Ic.grad, I64.grad, TOL_GRAD, "dI")
    _close(Pc.grad, P64.grad, TOL_GRAD, "dP")
    wrong = P64.grad.clone()
    wrong[-1] = 0                                                      # the last position's row dropped
    _far(Pc.grad, wrong, TOL_GRAD, "dP")


# --------------------------------------------------------------------------------------------------------------------
# residual LayerNorm
# --------------------------------------------------------------------------------------------------------------------

def _add_ln64(x, r, gamma, beta, unbiased=False):
    z = x + r
    mu = z.mean(-1, keepdim=True)
    var = ((z - mu) ** 2).sum(-1, keepdim=True) / (z.shape[-1] - (1 if unbiased else 0))
    return (z - mu) / torch.sqrt(var + 1e-5) * gamma + beta


@pytest.mark.parametrize("rows,d", [(1, 32), (4097, 32), (1, 64), (5000, 64), (1, 96), (4099, 96), (1, 128), (4100, 128),
                                    (1, 256), (4097, 256), (300, 256)])
def test_add_layernorm_matches_float64(rows, d):
    from rechorus_b200 import ops
    g = torch.Generator().manual_seed(rows * 7 + d)
    x, r, gy = (torch.randn(rows, d, generator=g) for _ in range(3))
    gam = 1 + 0.3 * torch.randn(d, generator=g)
    bet = 0.3 * torch.randn(d, generator=g)
    leaves = [t.double().requires_grad_(True) for t in (x, r, gam, bet)]
    ref = _add_ln64(*leaves)
    ref.backward(gy.double())
    cu = [t.cuda().requires_grad_(True) for t in (x, r, gam, bet)]
    y = ops.add_layernorm(cu[0].view(1, rows, d), cu[1].view(1, rows, d), cu[2], cu[3])
    y.backward(gy.cuda().view(1, rows, d))
    _close(y.view(rows, d), ref, TOL_OUT, "y")
    for name, a, b in zip(("dx", "dres", "dgamma", "dbeta"), cu, leaves):
        _close(a.grad, b.grad, TOL_GRAD, name)
    with torch.no_grad():
        _far(y.view(rows, d), _add_ln64(*(t.double() for t in (x, r, gam, bet)), unbiased=True), TOL_OUT, "y")


# --------------------------------------------------------------------------------------------------------------------
# whole models against the float64 oracle
# --------------------------------------------------------------------------------------------------------------------

# (emb_size, num_heads, num_layers, history_max); one-block models train only with the last-query block beyond L = 128
# or at d = 256, H = 8 (tests/test_seq_envelope_cpu.py checks that the others are refused)
MODEL_GRID = [(64, 4, 2, 128), (64, 4, 1, 200), (64, 4, 1, 256), (128, 4, 2, 86), (64, 1, 2, 100), (32, 1, 2, 128),
              (128, 2, 2, 64), (256, 8, 1, 50)]
MODEL_CASES = [(*c, lq) for c in MODEL_GRID for lq in (True, False) if lq or c[2] >= 2]


@pytest.mark.parametrize("d,H,layers,hm,lastq", MODEL_CASES)
def test_sasrec_matches_float64_oracle(monkeypatch, d, H, layers, hm, lastq):
    from rechorus_b200 import ops, plugin
    from rechorus_b200.runner import BaseRunner
    monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
    p = plugin.SASRec.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(["--emb_size", str(d), "--num_heads", str(H), "--num_layers", str(layers), "--history_max", str(hm),
                      "--num_neg", "4"])
    a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_unused.pt"
    B, C, n_items = 12, 5, 300
    torch.manual_seed(d + hm)
    m = plugin.SASRec(a, types.SimpleNamespace(n_users=10, n_items=n_items)).to(a.device)
    with torch.no_grad():
        for name, q in m.named_parameters():
            if "layer_norm" not in name:
                q.mul_(10.0)                                   # trained-scale weights: softmaxes far from uniform
    g = torch.Generator().manual_seed(d * 1000 + hm)
    lengths = torch.randint(1, hm + 1, (B,), generator=g)
    lengths[0], lengths[1] = hm, 1                             # the batch is as wide as history_max
    hist = torch.randint(1, n_items, (B, hm), generator=g) * (torch.arange(hm).view(1, hm) < lengths.view(B, 1))
    iid = torch.randint(1, n_items, (B, C), generator=g)
    batch = {"history_items": hist, "lengths": lengths, "item_id": iid}
    feed = {k: v.cuda() for k, v in batch.items()}
    feed.update(user_id=torch.zeros(B, dtype=torch.int64, device="cuda"), batch_size=B, phase="train")
    w64 = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    pred64, loss64, g64 = O.loss_and_grads("SASRec", w64, batch, H)
    m.train()
    out = m(feed)
    loss = m.loss(out)
    loss.backward()
    ops.check_ids()
    _close(out["prediction"], pred64, TOL_OUT, "prediction")
    _close(loss.view(1), loss64.view(1), TOL_OUT, "loss")
    names = [k for k, _ in m.named_parameters()]
    assert sorted(names) == sorted(g64)
    for k, prm in m.named_parameters():
        assert prm.grad is not None, k
        _close(prm.grad, g64[k], TOL_GRAD, k)
    m.eval()
    with torch.no_grad():
        _close(m(feed)["prediction"], pred64, TOL_OUT, "eval prediction")


# --------------------------------------------------------------------------------------------------------------------
# the construction-time query agrees with the launchers
# --------------------------------------------------------------------------------------------------------------------

AGREE_DH = [(32, 4), (64, 4), (64, 1), (96, 3), (128, 4), (128, 8), (128, 2), (256, 8), (256, 4), (288, 4)]
AGREE_L = [1, 44, 45, 47, 48, 84, 85, 86, 87, 114, 115, 128, 129, 256, 257]


def _runs(fn):
    """True when fn's launches are all accepted; False when a launcher refuses with B2R_E_UNSUPPORTED / B2R_E_BADARG"""
    from rechorus_b200.lib import B200RecError
    try:
        fn()
        torch.cuda.synchronize()
        return True
    except B200RecError as e:
        assert "(code -3)" in str(e) or "(code -1)" in str(e), str(e)
        return False


@pytest.mark.parametrize("d,H", AGREE_DH)
def test_seq_train_check_agrees_with_the_launchers(d, H):
    from rechorus_b200 import lib as Lb
    from rechorus_b200 import ops
    h = Lb.load()
    B = 2
    gam, bet = torch.ones(d, device="cuda"), torch.zeros(d, device="cuda")
    for L in AGREE_L:
        lengths = torch.tensor([L, 1], device="cuda")
        q, k, v = (torch.randn(B, L, d, device="cuda", requires_grad=True) for _ in range(3))
        ql = torch.randn(B, d, device="cuda", requires_grad=True)

        def layernorm(x):
            y = ops.add_layernorm(x, x.detach(), gam, bet)
            return y

        def full_block():
            ctx = ops.causal_attention(q, k, v, H, live=lengths)
            layernorm(ctx).sum().backward()

        def last_block():
            ctx = ops.attention_last(ql, k, v, lengths, H)
            layernorm(ctx).sum().backward()

        for verdict_args, fn in (((L, d, H, 1, 0), full_block), ((L, d, H, 0, Lb.SEQ_LAST_QUERY), last_block)):
            accepted = h.b2r_seq_train_check(*verdict_args) == 0
            assert _runs(fn) == accepted, (verdict_args, h.b2r_last_error().decode())
