"""GPU: the tensor-core Linear kernels -- k_linear_tc (forward, and dX through the transposed weight with the dropout
scale folded in) and k_linear_dw_tc + k_linear_dw_reduce (dW, dbias), with and without dropout -- against the float64
restatement and error model of tests/linear_tc_oracle.py, alone at the kernels' shape edges and inside one NeuMF
(config 3) and one SASRec (config 4) training step.

Every check is one of:
  * Tier A: operands whose splits, products and partial sums are all fp32 numbers; the kernel equals float64 exactly;
  * Tier B: |got - ref| <= gamma S + 2 * 2^-24 |ref| elementwise, gamma derived in the oracle for any summation order;
  * Tier C: max |got - ref| / S within the bar the oracle sets from H100 measurements (each ratio is recorded as a
    junit property);
  * routes: the library entry points each case runs and their return codes (a silent SGEMM fallback fails), and two
    runs giving the same bits.
"""
import numpy as np
import pytest
import torch

from tests import dropout_oracle as D
from tests import linear_tc_oracle as O

pytestmark = pytest.mark.gpu

SEED = 0x00C0FFEE12345678
ENTRIES = ("b2r_linear_fwd_tc", "b2r_linear_fwd_tc_dropout", "b2r_linear_fwd", "b2r_linear_fwd_dropout",
           "b2r_linear_tc", "b2r_linear_bwd_input",
           "b2r_linear_bwd_weight_tc", "b2r_linear_bwd_weight_tc_dropout", "b2r_linear_bwd_weight",
           "b2r_linear_bwd_weight_dropout")


def _dev():
    return torch.device("cuda", 0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture
def calls(monkeypatch):
    """(entry point, return code) of every Linear kernel call ops makes, in order"""
    from rechorus_b200 import lib as L
    h, rec = L.load(), []
    for n in ENTRIES:
        def wrap(*a, _fn=getattr(h, n), _n=n):
            rc = _fn(*a)
            rec.append((_n, rc))
            return rc
        monkeypatch.setattr(h, n, wrap)
    return rec


def _drop(p, site, step):
    from rechorus_b200 import ops
    st = ops.DropoutState(SEED, _dev())
    st.set(SEED, step)
    return ops.Drop(st.tick(), p, site)


def _keep(drop, M, N):
    """the keep mask of a NeuMF-style dropout site (row r, t = 0) from the snapshot the kernel read"""
    seed, step = (int(v) for v in drop.snapshot.cpu())
    m = D.dropout_mask(seed & 0xFFFFFFFFFFFFFFFF, step, drop.site, np.arange(M), np.zeros(M), N, drop.p)
    return torch.from_numpy(m).float()


def _exact(got, ref, what):
    """Tier A: the kernel's fp32 result is the float64 one (exactly representable, or one rounding of an exact product by
    the dropout scale)"""
    want = ref.float().cpu()
    got = got.cpu()
    if not torch.equal(got, want):
        bad = got != want
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError(f"{what}: Tier A: {int(bad.sum())} of {bad.numel()} elements differ from float64, first flat "
                             f"index {i}: {float(got.reshape(-1)[i])!r} != {float(want.reshape(-1)[i])!r}")


def _bc(kind, got, ref, S, gamma, what, record_property):
    """Tier B, then Tier C"""
    msg = O.bound_violation(got, ref, S, gamma)
    assert msg is None, f"{what}: Tier B (gamma {gamma:.3e}): {msg}"
    r = O.ratio(got, ref, S)
    record_property(f"ratio {kind} {what}", f"{r:.3e}")
    assert r <= O.TIER_C[kind], f"{what}: Tier C: max |err| / S = {r:.3e} > {O.TIER_C[kind]:.1e}"


def _trained(shape, g, scale):
    return torch.randn(shape, generator=g) * scale


# --------------------------------------------------------------------------------------------------------------------
# forward
# --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", O.fwd_grid(), ids=lambda c: f"M{c.M}-K{c.K}-N{c.N}-r{int(c.relu)}-b{int(c.bias)}-p{c.p}")
def test_forward_grid(case, calls, record_property):
    from rechorus_b200 import ops
    M, K, N = case.M, case.K, case.N
    drop = _drop(case.p, site=1, step=5) if case.p is not None else None
    keep = _keep(drop, M, N) if drop is not None else None
    s = drop.scale if drop is not None else 1.0

    def run(x, W, b):
        xc, Wc, bc = x.cuda(), W.cuda(), None if b is None else b.cuda()
        if drop is not None:
            return ops.linear_fwd_dropout(xc, Wc, bc, case.relu, drop, tc=True)
        return ops.linear_fwd_tc(xc, Wc, bc, case.relu)

    for lo_in in ("x", "w"):
        x, W, b = O.fwd_case_operands(case, lo_in)
        ref, _ = O.fwd_ref(x, W, b, case.relu, keep, s)
        _exact(run(x, W, b), ref, f"lo in {lo_in}")
    g = torch.Generator().manual_seed(M + 10 * K + 1000 * N)
    x, W = _trained((M, K), g, 2.0), _trained((N, K), g, 3.0 / K ** 0.5)
    b = _trained((N,), g, 0.5) if case.bias else None
    ref, S = O.fwd_ref(x, W, b, case.relu, keep, s)
    _bc("fwd", run(x, W, b), ref, S, O.gamma_fwd(K), "random", record_property)
    entry = "b2r_linear_fwd_tc_dropout" if drop is not None else "b2r_linear_fwd_tc"
    assert calls == [(entry, 0)] * 3, calls


# --------------------------------------------------------------------------------------------------------------------
# dX: ops.linear_bwd -> b2r_linear_tc with W^T (s W^T under dropout) and the ReLU mask
# --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", O.dx_grid(), ids=lambda c: f"M{c.M}-N{c.N}-K{c.K}-r{int(c.relu)}-p{c.p}")
def test_dx_grid(case, calls, record_property):
    from rechorus_b200 import ops
    M, N, K = case.M, case.N, case.K
    drop = _drop(case.p, site=0, step=7) if case.p is not None else None
    s = drop.scale if drop is not None else 1.0
    x = torch.empty(M, K, device=_dev())

    def run(dy, W, y):
        dx, dW, db = ops.linear_bwd(dy.cuda(), x, W.cuda(), None if y is None else y.cuda(), True, False, False, drop)
        assert dW is None and db is None
        return dx

    n = 0
    if s in (1.0, 2.0):                  # s W exact
        for lo_in in ("dy", "w"):
            dy, W, y = O.dx_case_operands(case, lo_in)
            ref, _ = O.dx_ref(dy, y, W, s)
            _exact(run(dy, W, y), ref, f"lo in {lo_in}")
            n += 1
    g = torch.Generator().manual_seed(M + 10 * K + 1000 * N + 1)
    dy, W = _trained((M, N), g, 0.3), _trained((N, K), g, 3.0 / N ** 0.5)
    y = _trained((M, N), g, 1.0).clamp_min(0) if case.relu else None
    ref, S = O.dx_ref(dy, y, W, s)
    _bc("dx", run(dy, W, y), ref, S, O.gamma_dx(N), "random", record_property)
    assert calls == [("b2r_linear_tc", 0)] * (n + 1), calls


# --------------------------------------------------------------------------------------------------------------------
# dW / dbias: ops.linear_bwd -> b2r_linear_bwd_weight_tc(_dropout)
# --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("case", O.dw_grid(), ids=lambda c: f"M{c.M}-N{c.N}-K{c.K}-r{int(c.relu)}-b{int(c.bias)}-p{c.p}")
def test_dw_grid(case, calls, record_property):
    from rechorus_b200 import ops
    M, N, K = case.M, case.N, case.K
    drop = _drop(case.p, site=2, step=9) if case.p is not None else None
    s = drop.scale if drop is not None else 1.0
    W = torch.empty(N, K, device=_dev())

    def run(dy, x, y):
        dx, dW, db = ops.linear_bwd(dy.cuda(), x.cuda(), W, None if y is None else y.cuda(), False, True, case.bias, drop)
        assert dx is None and (db is None) == (not case.bias)
        return dW, db

    operands = [("dense", O.dw_dense_operands(M, N, K))]
    operands += [(f"boundary rows, lo in {lo}", O.dw_sparse_operands(M, N, K, lo, _sms())) for lo in ("dy", "x")]
    for what, (dy, x, y) in operands:
        y = y if case.relu else None
        rW, _, rb, _ = O.dw_ref(dy, y, x, s)
        dW, db = run(dy, x, y)
        _exact(dW, rW, f"{what}: dW")
        if case.bias:
            _exact(db, rb, f"{what}: dbias")
    g = torch.Generator().manual_seed(M + 10 * K + 1000 * N + 2)
    dy, x = _trained((M, N), g, 0.3), _trained((M, K), g, 2.0)
    y = _trained((M, N), g, 1.0).clamp_min(0) if case.relu else None
    rW, SW, rb, Sb = O.dw_ref(dy, y, x, s)
    dW, db = run(dy, x, y)
    gamma = O.gamma_dw(M, _sms())
    _bc("dw", dW, rW, SW, gamma, "random dW", record_property)
    if case.bias:
        _bc("dw", db, rb, Sb, gamma, "random dbias", record_property)
    entry = "b2r_linear_bwd_weight_tc_dropout" if drop is not None else "b2r_linear_bwd_weight_tc"
    assert calls == [(entry, 0)] * 4, calls


@pytest.mark.parametrize("M", [1, 33, 255])
@pytest.mark.parametrize("N,K", [(4, 16), (68, 80), (128, 240)])
def test_dw_short_ranges_through_the_c_abi(M, N, K):
    """below ops' 4096-row threshold the C ABI still takes any M > 0: every row dense with lo bits, so the lo*hi / hi*lo
    products and the ones row carry exact values through ranges shorter than one 32-row slab"""
    from rechorus_b200 import lib as _lib
    L = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    ws = torch.empty(L.b2r_linear_bwd_weight_tc_workspace_bytes(M, N, K), dtype=torch.uint8, device=_dev())
    for lo_in in ("dy", "x"):
        dy, x, y = O.dw_small_operands(M, N, K, lo_in)
        for relu, p in ((False, None), (True, 0.5)):
            yy = y if relu else None
            s = D.dropout_scale(p) if p is not None else 1.0
            dyc, xc = dy.cuda(), x.cuda()
            yc = None if yy is None else yy.cuda()
            dW = torch.full((N, K), float("nan"), device=_dev())
            db = torch.full((N,), float("nan"), device=_dev())
            args = (dyc.data_ptr(), N, None if yc is None else yc.data_ptr(), xc.data_ptr(), K, dW.data_ptr(),
                    db.data_ptr(), M, N, K)
            if p is None:
                rc = L.b2r_linear_bwd_weight_tc(*args, ws.data_ptr(), ws.numel(), st)
            else:
                dc = _drop(p, site=0, step=1).c_struct()
                import ctypes
                rc = L.b2r_linear_bwd_weight_tc_dropout(*args, ctypes.byref(dc), ws.data_ptr(), ws.numel(), st)
            assert rc == 0
            rW, _, rb, _ = O.dw_ref(dy, yy, x, s)
            _exact(dW, rW, f"lo in {lo_in}, relu {relu}, p {p}: dW")
            _exact(db, rb, f"lo in {lo_in}, relu {relu}, p {p}: dbias")


# --------------------------------------------------------------------------------------------------------------------
# routes through ops.linear: threshold, misaligned views, column blocks, the dX class
# --------------------------------------------------------------------------------------------------------------------

def _route_check(x, W, b, relu, p, what):
    """forward + backward of ops.linear on x (any view); returns the calls' routes.  Checks y, dX, dW, db by Tier B with
    the gamma of the route each one took."""
    from rechorus_b200 import ops
    M, K = x.shape
    N = W.shape[0]
    drop = _drop(p, site=3, step=11) if p is not None else None
    s = drop.scale if drop is not None else 1.0
    xg = x.detach().requires_grad_(True)
    Wg, bg = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = ops.linear(xg, Wg, bg, relu=relu, drop=drop)
    g = torch.Generator().manual_seed(M + N + K)
    dy = _trained((M, N), g, 0.3).cuda()
    y.backward(dy)
    keep = _keep(drop, M, N) if drop is not None else None
    xc, Wc, bcpu = x.detach().cpu(), W.cpu(), b.cpu()
    ref, S = O.fwd_ref(xc, Wc, bcpu, relu, keep, s)
    yc = y.detach().cpu()
    tc = M >= 4096
    msg = O.bound_violation(yc, ref, S, O.gamma_fwd(K) if tc else O.gamma_sum(K + 1))
    assert msg is None, f"{what}: y: {msg}"
    rx, Sx = O.dx_ref(dy.cpu(), yc if relu else None, Wc, s)
    assert O.bound_violation(xg.grad.cpu(), rx, Sx, max(O.gamma_dx(N), O.gamma_sum(N) + O.U24)) is None, what
    rW, SW, rb, Sb = O.dw_ref(dy.cpu(), yc if relu else None, xc, s)
    gdw = max(O.gamma_dw(M, _sms()), O.gamma_sum(M))
    assert O.bound_violation(Wg.grad.cpu(), rW, SW, gdw) is None, what
    assert O.bound_violation(bg.grad.cpu(), rb, Sb, gdw) is None, what


def _misaligned(M, ld, K, g, scale=2.0):
    """an [M, K] view with row stride ld starting one float into its storage (not 16-byte aligned)"""
    buf = _trained((M * ld + 4,), g, scale).cuda()
    return buf[1:1 + M * ld].view(M, ld)[:, :K]


@pytest.mark.parametrize("p", [None, 0.3])
@pytest.mark.parametrize("M", [4095, 4096, 4097])
def test_routes_at_the_threshold(M, p, calls):
    g = torch.Generator().manual_seed(M)
    K, N = 64, 32
    x, W, b = _trained((M, K), g, 2.0).cuda(), _trained((N, K), g, 0.4).cuda(), _trained((N,), g, 0.5).cuda()
    _route_check(x, W, b, True, p, f"M={M}")
    d = "_dropout" if p is not None else ""
    if M >= 4096:
        want = [(f"b2r_linear_fwd_tc{d}", 0), ("b2r_linear_tc", 0), (f"b2r_linear_bwd_weight_tc{d}", 0)]
    else:
        want = [(f"b2r_linear_fwd{d}", 0), ("b2r_linear_bwd_input", 0), (f"b2r_linear_bwd_weight{d}", 0)]
    assert sorted(calls) == sorted(want), calls


@pytest.mark.parametrize("p", [None, 0.5])
def test_misaligned_views_are_refused_and_fall_back(p, calls, record_property):
    """x one float into its storage with ldx % 4 == 0: the forward and dW kernels refuse it (-3) and the SGEMM gives the
    result; dX reads only dY and W^T and stays on the tensor cores"""
    g = torch.Generator().manual_seed(5)
    M, K, N = 4160, 64, 64
    x = _misaligned(M, K + 4, K, g)
    assert x.data_ptr() % 16 != 0 and x.stride(0) % 4 == 0
    W, b = _trained((N, K), g, 0.4).cuda(), _trained((N,), g, 0.5).cuda()
    from rechorus_b200 import ops
    drop = _drop(p, site=3, step=11) if p is not None else None
    xg = x.detach().requires_grad_(True)
    Wg, bg = W.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = ops.linear(xg, Wg, bg, relu=True, drop=drop)
    dy = _trained((M, N), g, 0.3).cuda()
    y.backward(dy)
    d = "_dropout" if p is not None else ""
    assert calls == [(f"b2r_linear_fwd_tc{d}", -3), (f"b2r_linear_fwd{d}", 0), ("b2r_linear_tc", 0),
                     (f"b2r_linear_bwd_weight_tc{d}", -3), (f"b2r_linear_bwd_weight{d}", 0)], calls
    s = drop.scale if drop is not None else 1.0
    keep = _keep(drop, M, N) if drop is not None else None
    xc = x.detach().cpu()
    ref, S = O.fwd_ref(xc, W.cpu(), b.cpu(), True, keep, s)
    yc = y.detach().cpu()
    assert O.bound_violation(yc, ref, S, O.gamma_sum(K + 1)) is None
    rx, Sx = O.dx_ref(dy.cpu(), yc, W.cpu(), s)
    _bc("dx", xg.grad, rx, Sx, O.gamma_dx(N), "misaligned x: dX", record_property)
    rW, SW, rb, Sb = O.dw_ref(dy.cpu(), yc, xc, s)
    assert O.bound_violation(Wg.grad.cpu(), rW, SW, O.gamma_sum(M)) is None
    assert O.bound_violation(bg.grad.cpu(), rb, Sb, O.gamma_sum(M)) is None


def test_misaligned_dy_falls_back_for_dx_and_dw(calls):
    from rechorus_b200 import ops
    g = torch.Generator().manual_seed(6)
    M, K, N = 4096, 64, 64
    dy = _misaligned(M, N + 4, N, g, 0.3)
    x, W = _trained((M, K), g, 2.0).cuda(), _trained((N, K), g, 0.4).cuda()
    y = _trained((M, N), g, 1.0).clamp_min(0).cuda()
    y = torch.empty(M, N + 4, device=_dev())[:, :N].copy_(y)          # the saved output shares dY's row stride
    dx, dW, db = ops.linear_bwd(dy, x, W, y, True, True, True)
    assert calls == [("b2r_linear_tc", -3), ("b2r_linear_bwd_input", 0), ("b2r_linear_bwd_weight_tc", -3),
                     ("b2r_linear_bwd_weight", 0)], calls
    rx, Sx = O.dx_ref(dy.cpu(), y.cpu(), W.cpu())
    assert O.bound_violation(dx.cpu(), rx, Sx, O.gamma_sum(N)) is None
    rW, SW, rb, Sb = O.dw_ref(dy.cpu(), y.cpu(), x.cpu())
    assert O.bound_violation(dW.cpu(), rW, SW, O.gamma_sum(M)) is None
    assert O.bound_violation(db.cpu(), rb, Sb, O.gamma_sum(M)) is None


def test_column_block_of_a_wider_matrix(calls):
    """ldx > K: x is columns 64..127 of a 256-wide matrix (16-byte aligned): forward, dX and dW on the tensor cores"""
    g = torch.Generator().manual_seed(7)
    M, K, N = 8192, 64, 64
    x = _trained((M, 256), g, 2.0).cuda()[:, 64:64 + K]
    W, b = _trained((N, K), g, 0.4).cuda(), _trained((N,), g, 0.5).cuda()
    _route_check(x, W, b, False, None, "column block")
    assert calls == [("b2r_linear_fwd_tc", 0), ("b2r_linear_tc", 0), ("b2r_linear_bwd_weight_tc", 0)], calls


@pytest.mark.parametrize("N,K,tc", [(128, 192, False), (96, 256, False), (64, 256, True), (128, 128, True),
                                    (32, 240, True), (16, 64, False)])
def test_dx_route_follows_the_kernel_class(N, K, tc, calls):
    """linear_bwd asks the library whether k_linear_tc takes K output columns over a reduction of N: K in (128, 256]
    with N > 64 goes straight to the SGEMM, with no refused tensor-core call"""
    from rechorus_b200 import ops
    g = torch.Generator().manual_seed(N + K)
    M = 4096
    dy, W = _trained((M, N), g, 0.3).cuda(), _trained((N, K), g, 0.2).cuda()
    y = _trained((M, N), g, 1.0).clamp_min(0).cuda()
    dx, _, _ = ops.linear_bwd(dy, torch.empty(M, K, device=_dev()), W, y, True, False, False)
    assert calls == [("b2r_linear_tc" if tc else "b2r_linear_bwd_input", 0)], calls
    rx, Sx = O.dx_ref(dy.cpu(), y.cpu(), W.cpu())
    assert O.bound_violation(dx.cpu(), rx, Sx, O.gamma_dx(N) if tc else O.gamma_sum(N)) is None


# --------------------------------------------------------------------------------------------------------------------
# bit reproducibility at a SASRec step's size
# --------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("p", [None, 0.3])
def test_two_runs_give_the_same_bits(p, calls):
    from rechorus_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(8)
    M, K, N = 204800, 64, 64
    x = torch.randn(M, K, device="cuda", generator=g)
    W, b = torch.randn(N, K, device="cuda", generator=g) * 0.2, torch.randn(N, device="cuda", generator=g)
    dy = torch.randn(M, N, device="cuda", generator=g)
    drop = _drop(p, site=0, step=2) if p is not None else None

    def once():
        y = ops.linear_fwd_dropout(x, W, b, True, drop, tc=True) if drop is not None else ops.linear_fwd_tc(x, W, b, True)
        dx, dW, db = ops.linear_bwd(dy, x, W, y, True, True, True, drop)
        return [t.view(torch.int32).clone() for t in (y, dx, dW, db)]

    a, c = once(), once()
    for name, u, v in zip(("y", "dX", "dW", "db"), a, c):
        assert torch.equal(u, v), name
    d = "_dropout" if p is not None else ""
    assert calls == [(f"b2r_linear_fwd_tc{d}", 0), ("b2r_linear_tc", 0), (f"b2r_linear_bwd_weight_tc{d}", 0)] * 2


# --------------------------------------------------------------------------------------------------------------------
# in-model replay: every ops.linear call of one NeuMF (config 3) and one SASRec (config 4) training step
# --------------------------------------------------------------------------------------------------------------------

class _Recorder:
    """wraps ops.linear and ops.linear_bwd: the fp32 inputs and outputs of every call and the kernels each one ran"""

    def __init__(self, monkeypatch, calls):
        from rechorus_b200 import ops
        self.fwd, self.bwd = [], []
        linear, linear_bwd = ops.linear, ops.linear_bwd

        def rec_linear(x, W, bias=None, relu=False, drop=None):
            n0 = len(calls)
            y = linear(x, W, bias, relu, drop)
            K, N = W.shape[1], W.shape[0]
            self.fwd.append(dict(x=x.detach().reshape(-1, K).clone(), W=W.detach().clone(),
                                 b=None if bias is None else bias.detach().clone(), relu=relu, drop=drop,
                                 y=y.detach().reshape(-1, N).clone(), routes=list(calls[n0:])))
            return y

        def rec_bwd(dy, x, W, y_relu, need_dx, need_dw, need_db, drop=None):
            n0 = len(calls)
            dx, dW, db = linear_bwd(dy, x, W, y_relu, need_dx, need_dw, need_db, drop)
            self.bwd.append(dict(dy=dy.detach().clone(), x=x.detach().clone(), W=W.detach(), y=y_relu, drop=drop,
                                 dx=dx, dW=dW, db=db, routes=list(calls[n0:])))
            return dx, dW, db

        monkeypatch.setattr(ops, "linear", rec_linear)
        monkeypatch.setattr(ops, "linear_bwd", rec_bwd)


def _build(name, extra, n_users, n_items):
    import argparse
    import types
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    a = cls.parse_model_args(p).parse_args(extra)
    a.device, a.model_path = _dev(), "/tmp/_b2r_unused.pt"
    torch.manual_seed(0)
    m = cls(a, types.SimpleNamespace(n_users=n_users, n_items=n_items)).to(a.device)
    with torch.no_grad():
        for n_, q in m.named_parameters():
            if "layer_norm" not in n_:
                q.mul_(10.0)                      # trained-scale weights
    m.train()
    return m


def _check_records(rec, device, record_property):
    """Tier B and C of every recorded call against float64 on ``device``, gamma from the route it took"""
    for i, r in enumerate(rec.fwd):
        x, W, drop = r["x"], r["W"], r["drop"]
        M, K = x.shape
        N = W.shape[0]
        keep = _keep(drop, M, N).to(device) if drop is not None else None
        s = drop.scale if drop is not None else 1.0
        ref, S = O.fwd_ref(x, W, r["b"], r["relu"], keep, s, device)
        tc = r["routes"][-1][0].startswith("b2r_linear_fwd_tc")
        _bc("fwd", r["y"], ref, S, O.gamma_fwd(K) if tc else O.gamma_sum(K + 1), f"forward {i} M{M} K{K} N{N}",
            record_property)
    sms = _sms()
    for i, r in enumerate(rec.bwd):
        dy, x, W, y, drop = r["dy"], r["x"], r["W"], r["y"], r["drop"]
        M, N = dy.shape
        K = W.shape[1]
        s = drop.scale if drop is not None else 1.0
        names = [n for n, _ in r["routes"]]
        what = f"backward {i} M{M} N{N} K{K}"
        if r["dx"] is not None:
            ref, S = O.dx_ref(dy, y, W, s, device)
            gamma = O.gamma_dx(N) if "b2r_linear_tc" in names else O.gamma_sum(N) + O.U24
            _bc("dx", r["dx"], ref, S, gamma, what + " dX", record_property)
        rW, SW, rb, Sb = O.dw_ref(dy, y, x, s, device)
        gamma = O.gamma_dw(M, sms) if any(n.startswith("b2r_linear_bwd_weight_tc") for n in names) else O.gamma_sum(M)
        _bc("dw", r["dW"], rW, SW, gamma, what + " dW", record_property)
        if r["db"] is not None:
            _bc("dw", r["db"], rb, Sb, gamma, what + " dbias", record_property)


def _by_weight(rec, model):
    """recorded backward calls keyed by the parameter (and column offset) their W is"""
    out = {}
    params = dict(model.named_parameters())
    for r in rec.bwd:
        for name, q in params.items():
            off = (r["W"].data_ptr() - q.data_ptr()) // 4
            if q.dim() == 2 and 0 <= off < q.shape[1] and r["W"].shape[0] == q.shape[0]:
                out[name] = (r, off)
    return out


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("dropout", [0.0, 0.2])
def test_neumf_config3_step_replay(dropout, monkeypatch, calls, record_property):
    """NeuMF, d = 64, layers [64, 32, 16], B = 4096, C = 5 (20,480 rows): the hidden layers' forward, dX (except the
    16-wide last layer's) and dW on the tensor cores, the 1-wide prediction layer on the SGEMM"""
    rec = _Recorder(monkeypatch, calls)
    n = 20000
    m = _build("NeuMF", ["--emb_size", "64", "--layers", "[64, 32, 16]", "--num_neg", "4", "--dropout", str(dropout)],
               n, n)
    g = torch.Generator().manual_seed(3)
    B, C = 4096, 5
    feed = {"user_id": torch.randint(1, n, (B,), generator=g).cuda(), "item_id": torch.randint(1, n, (B, C), generator=g).cuda(),
            "batch_size": B, "phase": "train"}
    m.loss(m(feed)).backward()
    torch.cuda.synchronize()
    d = "_dropout" if dropout > 0 else ""
    assert [r["routes"] for r in rec.fwd] == [[(f"b2r_linear_fwd_tc{d}", 0)]] * 3 + [[("b2r_linear_fwd", 0)]]
    assert [r["x"].shape[0] for r in rec.fwd] == [B * C] * 4
    want = {"mlp.0.weight": [("b2r_linear_tc", 0), (f"b2r_linear_bwd_weight_tc{d}", 0)],
            "mlp.1.weight": [("b2r_linear_tc", 0), (f"b2r_linear_bwd_weight_tc{d}", 0)],
            "mlp.2.weight": [("b2r_linear_bwd_input", 0), (f"b2r_linear_bwd_weight_tc{d}", 0)],
            "prediction.weight": [("b2r_linear_bwd_input", 0), ("b2r_linear_bwd_weight", 0)]}
    byw = _by_weight(rec, m)
    assert sorted(byw) == sorted(want) and len(rec.bwd) == 4
    params = dict(m.named_parameters())
    for name, routes in want.items():
        r, off = byw[name]
        assert r["routes"] == routes, (name, r["routes"])
        grad = params[name].grad
        assert _bits(grad[:, off:off + r["dW"].shape[1]], r["dW"]), name
        if name.startswith("mlp."):
            assert _bits(params[name.replace("weight", "bias")].grad, r["db"]), name
    _check_records(rec, "cpu", record_property)


def test_sasrec_config4_step_replay(monkeypatch, calls, record_property):
    """SASRec, d = 64, 2 blocks, 4 heads, B = 4096, L = 50, last-query block: block 0's five Linears and block 1's k / v
    over 204,800 rows and block 1's q / linear1 / linear2 over the 4,096 last-query rows, all on the tensor cores
    (float64 reference on the GPU: the CPU would take minutes over the 204,800-row calls)"""
    rec = _Recorder(monkeypatch, calls)
    n_items = 20000
    m = _build("SASRec", ["--emb_size", "64", "--history_max", "50", "--num_layers", "2", "--num_heads", "4",
                          "--num_neg", "99"], 10, n_items)
    B, C, L = 4096, 100, 50
    g = torch.Generator().manual_seed(4)
    lengths = torch.randint(1, L + 1, (B,), generator=g)
    lengths[0] = L
    hist = torch.randint(1, n_items, (B, L), generator=g) * (torch.arange(L).view(1, L) < lengths.view(B, 1))
    feed = {"user_id": torch.zeros(B, dtype=torch.int64).cuda(), "item_id": torch.randint(1, n_items, (B, C), generator=g).cuda(),
            "history_items": hist.cuda(), "lengths": lengths.cuda(), "batch_size": B, "phase": "train"}
    m.loss(m(feed)).backward()
    torch.cuda.synchronize()
    assert all(r["routes"] == [("b2r_linear_fwd_tc", 0)] for r in rec.fwd), [r["routes"] for r in rec.fwd]
    assert sorted(r["x"].shape[0] for r in rec.fwd) == [B] * 3 + [B * L] * 7
    assert len(rec.bwd) == 10
    assert all(r["routes"] == [("b2r_linear_tc", 0), ("b2r_linear_bwd_weight_tc", 0)] for r in rec.bwd), \
        [r["routes"] for r in rec.bwd]
    byw = _by_weight(rec, m)
    assert len(byw) == 10
    params = dict(m.named_parameters())
    for name, (r, _) in byw.items():
        assert _bits(params[name].grad, r["dW"]), name
        assert _bits(params[name.replace("weight", "bias")].grad, r["db"]), name
    _check_records(rec, "cuda", record_property)
