"""The first half of every BPR training step against float64 (tests/bpr_oracle.py): candidate scoring, the BPR loss and
the query-side gradient dQ, on k_bprmf_flash (the whole-step route), the unfused rowdot / loss / rowdot_bwd_query
kernels (the contract route and the step's fallback) and the shard owner's pairdot / pair_runs_sum.

Scores are checked bit for bit on exact operands (Tier A) and within gamma_dot Sabs otherwise; loss, g and dQ within
the error model's bounds evaluated on each kernel's own float32 pred (Tier B), over the kernels' shape edges and the
score regimes that stress the softmax and the clamp window; Tier C bars on the well-conditioned cases."""
import math

import numpy as np
import pytest
import torch

from tests import bpr_oracle as O
from tests import table_grad_oracle as TG

pytestmark = pytest.mark.gpu

RATIOS = {k: 0.0 for k in O.TIER_C}


def _dev():
    return torch.device("cuda", 0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _flag():
    from rechorus_b200 import ops
    return int(ops.err_flag(_dev()).item())


def _clear_flag():
    from rechorus_b200 import ops
    ops.err_flag(_dev()).zero_()


def _note(what, r):
    RATIOS[what] = max(RATIOS[what], r)


def _exact_case(regime, B, C, d, seed=0):
    g = torch.Generator().manual_seed(seed * 7919 + B * 131 + C * 17 + d + O.REGIMES.index(regime))
    U, T, ids = O.exact_operands(O.regime_targets(regime, B, C, g), d, g)
    if regime == "dup":
        ids = O.add_duplicates(ids, g)
    return U.to(_dev()), T.to(_dev()), ids.to(_dev())


def _bpr_loss_rows(pred):
    """b2r_bpr_loss with its per-row losses: (loss, g, row_loss)"""
    from rechorus_b200 import lib as L_, ops
    B, Cn = pred.shape
    loss = torch.empty((), dtype=torch.float32, device=pred.device)
    g = torch.empty_like(pred)
    rows = torch.empty(B, dtype=torch.float32, device=pred.device)
    L_.check(L_.load().b2r_bpr_loss(ops._p(pred), ops._p(loss), ops._p(g), ops._p(rows), B, Cn, ops._stream()),
             "b2r_bpr_loss")
    return loss, g, rows


# ------------------------------------------------------------------------------------------------------------------
# a. k_bprmf_flash through ops.bprmf_fused_fwd_bwd
# ------------------------------------------------------------------------------------------------------------------

def _flash_cases():
    """per d: C - 1 at the chunk edges (1; GPW - 1: the last lane group gets no negative; GPW: one each; 512/d - 1,
    512/d, 512/d + 1; 2 (512/d) + 1: the two-chunk prologue; 1023: C = 1024, the kernel's limit) and C = 1, with B and
    the score regime rotating; then every regime at one mid shape per d"""
    out, i = [], 0
    bs = (7, 1, 4096)
    for d in (32, 64, 128):
        k, G = 512 // d, 128 // d
        for cm1 in sorted({0, 1, G - 1, G, k - 1, k, k + 1, 2 * k + 1, 1023}):
            B = bs[i % 3] if cm1 < 1023 else (7, 1)[i % 2]
            out.append((d, cm1 + 1, B, O.REGIMES[i % len(O.REGIMES)]))
            i += 1
        for regime in O.REGIMES:
            out.append((d, 100, 64, regime))
    return out


def _check_flash(d, C, B, regime, U, T, ids, uid=None):
    from rechorus_b200 import ops
    uid = torch.arange(B, device=_dev()) if uid is None else uid
    f0 = _flag()
    pred, gp, rl, dq = ops.bprmf_fused_fwd_bwd(U, uid, T, ids)
    ref, _ = O.score_ref(U, uid, T, ids)
    assert torch.equal(pred.double(), ref), "Tier A: pred must equal float64"
    assert torch.equal(pred, ops.rowdot(U, uid, T, ids)), "pred must carry k_rowdot_fwd's bits"
    assert _flag() == f0
    L = O.loss_ref(pred, "flash", d)
    assert O.ambiguity_ok(L, regime) is None, O.ambiguity_ok(L, regime)
    for msg in (O.loss_violation(rl, L), O.g_violation(gp, L)):
        assert msg is None, msg
    dqr = O.dq_ref(L.g_in, T, ids)
    bf = O.dq_bound_flash(L, T, ids, d)
    msg = O.dq_violation(dq, dqr, bf, L)
    assert msg is None, msg
    if regime == "below" or C == 1:
        assert bool((gp == 0).all()) and bool((dq == 0).all())
    if C == 1:
        assert torch.equal(rl, torch.full_like(rl, rl[0].item())) and abs(rl[0].item() + math.log(O.LO)) < 4e-6
    # cross-route: loss.cu + rowdot_bwd_query on the same pred, within the sum of the two bounds
    Ls = O.loss_ref(pred, "loss")
    _, gs, rs = _bpr_loss_rows(pred)
    for msg in (O.loss_violation(rs, Ls), O.g_violation(gs, Ls)):
        assert msg is None, msg
    dqs = ops.rowdot_bwd_query(gs, T, ids)
    bs = O.dq_bound_sep(Ls, T, ids, d)
    msg = O.dq_violation(dqs, dqr, bs, Ls)
    assert msg is None, msg
    both = ~(L.ambiguous | Ls.ambiguous)
    assert bool(((gp.double() - gs.double()).abs() <= L.err_g + Ls.err_g)[both].all())
    assert bool(((dq.double() - dqs.double()).abs() <= bf + bs)[both].all())
    if regime in O.WELL_CONDITIONED and C > 1:
        _note("g", O.worst_ratio(gp, L.g_in, L.g_scale))
        _note("dq", O.worst_ratio(dq, dqr, O.dq_scale(L, T, ids)))
        if C >= 3:          # the wrong references fall outside the bounds on these cases
            for v in ("detached", "pos_in_softmax", "mean_bc", "sig_flipped"):
                assert O.wrong_ratio(O.wrong_g(pred, v), L, L.err_g) > 1, v
            assert O.dq_violation(O.wrong_dq_no_g0r0(L, T, ids), dqr, bf, L) is not None
    if regime == "below" and C > 1:
        assert O.wrong_ratio(O.wrong_g(pred, "no_clamp"), L, L.err_g) > 1
    return pred, gp, rl, dq


@pytest.mark.parametrize("d,C,B,regime", _flash_cases())
def test_flash_kernel_vs_float64(d, C, B, regime):
    U, T, ids = _exact_case(regime, B, C, d)
    _check_flash(d, C, B, regime, U, T, ids)


@pytest.mark.parametrize("d", [32, 128])
def test_flash_kernel_past_resident_cap(d):
    """B one sample past sm_count x 32 CTAs x 8 warps: warps loop over samples and reuse their ring, sid[] and xs[]"""
    B = 8 * 32 * _sms() + 1
    U, T, ids = _exact_case("trained", B, 512 // d + 1, d)
    _check_flash(d, 512 // d + 1, B, "trained", U, T, ids)


def test_flash_kernel_out_of_range_ids_clamped_and_counted():
    from rechorus_b200 import ops
    d, B, C = 64, 9, 20
    U, T, ids = _exact_case("well", B, C, d)
    ids = ids.clone()
    ids[0, 3], ids[4, 0], ids[8, 19] = -1, T.shape[0] + 5, T.shape[0]
    uid = torch.arange(B, device=_dev())
    uid[2] = -4
    _clear_flag()
    pred, gp, rl, dq = ops.bprmf_fused_fwd_bwd(U, uid, T, ids)
    assert _flag() == 4                                   # three candidate ids, one user id: counted once each
    _clear_flag()
    ref, _ = O.score_ref(U, uid, T, ids)                  # clamped to row 0
    assert torch.equal(pred.double(), ref)
    L = O.loss_ref(pred, "flash", d)
    assert O.g_violation(gp, L) is None
    assert O.dq_violation(dq, O.dq_ref(L.g_in, T, ids), O.dq_bound_flash(L, T, ids, d), L) is None
    with pytest.raises(IndexError):
        ops.rowdot(U, uid, T, ids)
        ops.check_ids()
    _clear_flag()


def test_flash_kernel_is_deterministic():
    from rechorus_b200 import ops
    for d in (32, 64, 128):
        U, T, ids = _exact_case("asc", 300, 257, d)
        uid = torch.arange(300, device=_dev())
        a = ops.bprmf_fused_fwd_bwd(U, uid, T, ids)
        b = ops.bprmf_fused_fwd_bwd(U, uid, T, ids)
        for x, y in zip(a, b):
            assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------------------------
# b. the whole step through ops.bprmf_train_step
# ------------------------------------------------------------------------------------------------------------------

class _Tables(torch.nn.Module):
    def __init__(self, U, I):
        super().__init__()
        self.U = torch.nn.Parameter(U.clone())
        self.I = torch.nn.Parameter(I.clone())


def _step_model(U, I, lr):
    from rechorus_b200 import ops
    from rechorus_b200.optim import RowSparseOptimizer
    m = _Tables(U, I)
    for p in m.parameters():
        ops.set_table_mode(p, "fused")
    return m, RowSparseOptimizer(m, "SGD", lr=lr, l2=0.0)


def _check_item_update(I0, I1, uid, ids, g, U, lr):
    """moved item rows equal -lr sum g U[uid] within the table-gradient bound; the rest keep their bits"""
    B, C = ids.shape
    tg = TG.table_grad(ids, I0.shape[0], I0.shape[1], [TG.Stream(src=U[uid].contiguous(), n=B * C, ld=U.shape[1],
                                                                 coef=g.reshape(-1), div=C)])
    moved = I1.double()[tg.rows] - I0.double()[tg.rows]
    want = -lr * tg.grad
    bnd = lr * tg.bound() + 2 * O.u * (I1.double()[tg.rows].abs() + I0.double()[tg.rows].abs())
    bnd = bnd + 2.0 ** -149 * (tg.count + 2).unsqueeze(1)        # float32 subnormals: each rounding may lose 2^-150
    assert bool(((moved - want).abs() <= bnd).all())
    keep = torch.ones(I0.shape[0], dtype=torch.bool, device=I0.device)
    keep[tg.rows] = False
    assert torch.equal(I1[keep], I0[keep])


def test_train_step_loss_is_the_tree_mean_and_qout_feeds_the_item_update():
    from rechorus_b200 import ops
    d, B, C = 64, 1000, 33
    batches = [_exact_case(r, B, C, d, seed=s) for s, r in enumerate(("trained", "well", "dup"))]
    U, T, _ = batches[0]
    m, opt = _step_model(U, T, 0.0)
    uid = torch.arange(B, device=_dev())
    for t in range(2):                                    # the second step needs done_counter reset by the first
        _, _, ids = batches[t]
        loss = ops.bprmf_train_step(m.U, m.I, opt, uid, ids)
        _, _, rl, _ = ops.bprmf_fused_fwd_bwd(m.U.data, uid, m.I.data, ids)
        assert float(loss) == float(O.tree_mean_f32(rl.cpu().numpy(), 256)), t
        assert np.float32(loss.item()).tobytes() == O.tree_mean_f32(rl.cpu().numpy(), 256).tobytes()
    assert torch.equal(m.U.data, U) and torch.equal(m.I.data, T)
    lr = 0.5
    m, opt = _step_model(U, T, lr)
    _, _, ids = batches[2]
    _, gp, _, _ = ops.bprmf_fused_fwd_bwd(U, uid, T, ids)
    ops.bprmf_train_step(m.U, m.I, opt, uid, ids)
    _check_item_update(T, m.I.data, uid, ids, gp, U, lr)


def test_train_step_fallback_route_within_the_loss_bounds():
    """C = 1025 is past the streaming kernel's limit: gather / rowdot / loss.cu / rowdot_bwd_query"""
    from rechorus_b200 import ops
    d, B, C = 64, 40, 1025
    U, T, ids = _exact_case("spike", B, C, d)
    uid = torch.arange(B, device=_dev())
    m, opt = _step_model(U, T, 0.5)
    loss = ops.bprmf_train_step(m.U, m.I, opt, uid, ids)
    pred = ops.rowdot(U, uid, T, ids)
    l2, g, rows = _bpr_loss_rows(pred)
    assert float(loss) == float(l2) == float(O.tree_mean_f32(rows.cpu().numpy(), 1024))
    L = O.loss_ref(pred, "loss")
    assert O.loss_violation(rows, L) is None and O.g_violation(g, L) is None
    _check_item_update(T, m.I.data, uid, ids, g, U, 0.5)


# ------------------------------------------------------------------------------------------------------------------
# c. the unfused family
# ------------------------------------------------------------------------------------------------------------------

ALL_D = (4, 20, 32, 64, 96, 128, 256)
ALL_C = (1, 7, 8, 9, 64, 65, 1000)


def _rowdot_cases():
    out = []
    for i, d in enumerate(ALL_D):
        out.append((d, 5, ALL_C[i % 7]))
        out.append((d, 37, ALL_C[(i + 3) % 7]))
        out.append((d, 11000, 65))                       # past grid_for's 16 x sm_count CTAs at every d
    return out


@pytest.mark.parametrize("d,B,C", _rowdot_cases())
def test_rowdot_and_gather_vs_float64(d, B, C):
    from rechorus_b200 import ops
    g = torch.Generator(device=_dev()).manual_seed(d * 100 + C)
    Q = torch.randn(B + 3, d, device=_dev(), generator=g)
    T = torch.randn(997, d, device=_dev(), generator=g)
    qid = torch.randint(0, B + 3, (B,), device=_dev(), generator=g)
    ids = torch.randint(0, 997, (B, C), device=_dev(), generator=g)
    f0 = _flag()
    pred = ops.rowdot(Q, qid, T, ids)
    ref, Sabs = O.score_ref(Q, qid, T, ids)
    assert O.score_violation(pred, ref, Sabs, d) is None
    _note("score", O.worst_ratio(pred, ref, Sabs))
    q = ops.gather_rows(Q, qid)
    assert torch.equal(q, Q[qid])
    assert torch.equal(ops.rowdot(q, None, T, ids), pred)            # dense-Q form: the same bits
    assert _flag() == f0
    if B <= 40:                                                       # Tier A: exact operands, bit for bit
        ge = torch.Generator().manual_seed(d + C)
        Qe = (torch.randint(-8, 9, (B + 3, d), generator=ge).float() / 8).to(_dev())
        Te = (torch.randint(-8, 9, (997, d), generator=ge).float() / 8).to(_dev())
        assert O.exact_ok(Qe, qid, Te, ids) is None
        assert torch.equal(ops.rowdot(Qe, qid, Te, ids).double(), O.score_ref(Qe, qid, Te, ids)[0])


@pytest.mark.parametrize("d", ALL_D)
def test_gather_rows_strided_bit_exact(d):
    from rechorus_b200 import lib as L_, ops
    g = torch.Generator(device=_dev()).manual_seed(d)
    T = torch.randn(500, d, device=_dev(), generator=g)
    for n, out_ld, div in ((37, d, 1), (1003, d + 12, 3), (20000, 2 * d, 7)):
        ids = torch.randint(0, 500, (-(-n // div),), device=_dev(), generator=g)
        out = torch.full((n, out_ld), 7.5, device=_dev())
        L_.check(L_.load().b2r_gather_rows_strided(ops._p(T), ops._p(ids), 500, ops._p(out), out_ld, n, d, div,
                                                   ops._p(ops.err_flag(_dev())), ops._stream()), "gather_rows_strided")
        r = torch.arange(n, device=_dev()) // div
        assert torch.equal(out[:, :d], T[ids[r]])
        assert bool((out[:, d:] == 7.5).all())


def _bwd_cases():
    out = []
    for d in (32, 64, 128):
        gpc = 256 // (d // 4)
        for nchunk in (1, 2, 3, gpc, gpc + 1):
            out.append((d, 9, 8 * nchunk - (3 if nchunk > 1 else 0)))
        out.append((d, 70000, 8))                          # past 16 x sm_count CTAs of GPC / GPS samples
    for d in (4, 20, 96, 256):
        out += [(d, 9, 1), (d, 9, 65), (d, 20000, 7)]
    return out


@pytest.mark.parametrize("d,B,C", _bwd_cases())
def test_rowdot_bwd_query_vs_float64(d, B, C):
    from rechorus_b200 import ops
    g = torch.Generator(device=_dev()).manual_seed(d * 1000 + C)
    T = torch.randn(999, d, device=_dev(), generator=g)
    ids = torch.randint(0, 999, (B, C), device=_dev(), generator=g)
    gp = torch.randn(B, C, device=_dev(), generator=g)
    dq = ops.rowdot_bwd_query(gp, T, ids)
    R = T.double()[ids]
    ref = torch.einsum("bc,bcd->bd", gp.double(), R)
    S = torch.einsum("bc,bcd->bd", gp.double().abs(), R.abs())
    assert O._violation(dq, ref, O.gamma(O.n_bwd(C, d)) * S, "dQ") is None


def _loss_cases():
    out, i = [], 0
    for B, C in ((8, 2), (9, 32), (1025, 33), (100000, 2), (100000, 32), (8, 1025), (9, 5000), (1025, 1025),
                 (64, 100), (33, 1), (300, 64), (4096, 100)):
        out.append((B, C, O.REGIMES[i % len(O.REGIMES)]))
        i += 1
    for regime in O.REGIMES:
        out.append((257, 129, regime))
    return out


@pytest.mark.parametrize("B,C,regime", _loss_cases())
def test_bpr_loss_kernel_vs_float64(B, C, regime):
    from rechorus_b200 import ops
    g = torch.Generator().manual_seed(B * 31 + C)
    pred = O.regime_targets(regime, B, C, g).float().to(_dev())
    loss, gp, rows = _bpr_loss_rows(pred)
    L = O.loss_ref(pred, "loss")
    assert O.ambiguity_ok(L, regime) is None, O.ambiguity_ok(L, regime)
    for msg in (O.loss_violation(rows, L), O.g_violation(gp, L)):
        assert msg is None, msg
    assert np.float32(loss.item()).tobytes() == O.tree_mean_f32(rows.cpu().numpy(), 1024).tobytes()
    if regime == "below":
        assert bool((gp == 0).all())
    if regime in O.WELL_CONDITIONED and C > 1:
        _note("g", O.worst_ratio(gp, L.g_in, L.g_scale))
    l2, g2 = ops.bpr_loss_and_grad(pred)
    assert torch.equal(l2, loss) and torch.equal(g2, gp)
    p = pred.clone().requires_grad_(True)                 # autograd node: value, and gradient times the upstream factor
    (ops.bpr_loss(p) * 2.0).backward()
    assert torch.equal(p.grad, 2 * gp)


# ------------------------------------------------------------------------------------------------------------------
# d. the shard owner's side
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [32, 64, 128, 20, 96])
def test_pairdot_and_p2p_vs_float64(d):
    from rechorus_b200 import ops
    g = torch.Generator(device=_dev()).manual_seed(d)
    for n in (5, 4099, 600000):
        Q = torch.randn(300, d, device=_dev(), generator=g)
        T = torch.randn(777, d, device=_dev(), generator=g)
        qidx = torch.randint(0, 300, (n,), device=_dev(), generator=g)
        rows = torch.randint(-200, 777, (n,), device=_dev(), generator=g).clamp_min(-1)   # ~20 % unused slots
        out = ops.pairdot(Q, qidx, T, rows)
        ref, Sabs = O.pair_ref(Q, qidx, T, rows)
        assert O.score_violation(out, ref, Sabs, d) is None
        assert bool((out[rows < 0] == 0).all())
        _note("score", O.worst_ratio(out, ref, Sabs))
        if d in (32, 64, 128):
            nseg = 4 if n % 4 == 0 else 1
            seg = n // nseg
            bufs = [torch.full((seg,), -3.0, device=_dev()) for _ in range(nseg)]
            tab = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=_dev())
            ops.pairdot_p2p(Q, qidx, T, rows, tab, seg)
            assert torch.equal(torch.cat(bufs), out)
        if n == 4099:                                      # Tier A
            ge = torch.Generator().manual_seed(d)
            Qe = (torch.randint(-8, 9, (300, d), generator=ge).float() / 8).to(_dev())
            Te = (torch.randint(-8, 9, (777, d), generator=ge).float() / 8).to(_dev())
            assert torch.equal(ops.pairdot(Qe, qidx, Te, rows).double(), O.pair_ref(Qe, qidx, Te, rows)[0])


@pytest.mark.parametrize("d", [32, 64, 128])
@pytest.mark.parametrize("big", [False, True])
def test_pair_runs_sum_vs_float64(d, big):
    """runs of 1, LPR - 1, LPR, LPR + 1 and 3 LPR + 5 elements from every offset inside a block, invalid slots and
    out-of-range keys between them, n % LPR != 0; big: past the grid cap (16 x sm_count CTAs), random run lengths"""
    from rechorus_b200 import ops
    lpr = d // 4
    n_out = 200000 if big else 400
    key, rows, coef, nk = O.runs_case(lpr, d + big, n_out=n_out, n_min=700000 if big else 0)
    g = torch.Generator(device=_dev()).manual_seed(d)
    T = torch.randn(50, d, device=_dev(), generator=g)
    out0 = torch.randn(n_out, d, device=_dev(), generator=g)
    key, rows, coef = key.to(_dev()), rows.to(_dev()), coef.to(_dev())
    out = out0.clone()
    ops.pair_runs_sum(out, key, rows, coef, T)
    ref, bnd = O.pair_runs_ref(out0, key, rows, coef, T)
    assert O._violation(out, ref, bnd, "pair_runs") is None
    assert torch.equal(out[nk:], out0[nk:])                               # rows no run targets keep their bits
    R = T.double()[rows.clamp_min(0)]
    scale = torch.zeros_like(ref).index_add_(0, key.clamp(0, n_out - 1),
                                             (coef.double().abs().unsqueeze(1) * R.abs()) * ((rows >= 0) & (key >= 0)
                                                                                             & (key < n_out)).unsqueeze(1))
    _note("pair_runs", O.worst_ratio(out, ref, scale))
    for v in ("cut", "skip_head"):                                         # the wrong references fall outside
        bad, _ = O.pair_runs_ref(out0, key, rows, coef, T, variant=v, lpr=lpr)
        assert O._violation(bad, ref, bnd, v) is not None
    # Tier A: coefficients and rows on the 2^-3 grid -> every partial sum exact
    ge = torch.Generator().manual_seed(d)
    ce = (torch.randint(-8, 9, (key.numel(),), generator=ge).float() / 8).to(_dev())
    Te = (torch.randint(-8, 9, (50, d), generator=ge).float() / 8).to(_dev())
    out = out0.clone()
    ops.pair_runs_sum(out, key, rows, ce, Te)
    assert torch.equal(out.double(), O.pair_runs_ref(out0, key, rows, ce, Te)[0])


# ------------------------------------------------------------------------------------------------------------------
# e. Tier C
# ------------------------------------------------------------------------------------------------------------------

def test_zz_tier_c_accuracy_bars():
    """worst max |got - ref| / scale over the well-conditioned cases above (run with the rest of the file)"""
    print("\nTier C worst ratios:", {k: f"{v:.3e}" for k, v in RATIOS.items()})
    for k, v in RATIOS.items():
        assert v <= O.TIER_C[k], (k, v, O.TIER_C[k])
