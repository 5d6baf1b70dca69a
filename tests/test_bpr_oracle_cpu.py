"""CPU checks of tests/bpr_oracle.py: the float32 emulations of k_bprmf_flash and k_bpr_loss_rows, with every exp,
divide and log moved to the edge of its documented error, stay inside the bounds in every score regime of the GPU
suite; the bounds are tight where conditioning allows; every deliberately wrong reference falls outside them by at
least 10x; the float32 tree means and the pair-run reference match hand-made cases.  No GPU needed."""
import math

import numpy as np
import pytest
import torch

from tests import bpr_oracle as O

DS = (32, 64, 128)


def _case(regime, B, C, d, seed=0):
    """(Q [B, d], R [B, C, d]) float32 with exact scores at the regime's targets (Tier A operands)"""
    g = torch.Generator().manual_seed(seed * 7919 + B * 131 + C * 17 + d + O.REGIMES.index(regime))
    tgt = O.regime_targets(regime, B, C, g)
    U, T, ids = O.exact_operands(tgt, d, g)
    if regime == "dup":
        ids = O.add_duplicates(ids, g)
    return U, T, ids


def _rows(U, T, ids):
    return U.numpy(), T[ids].numpy()


def _c_edges(d):
    k = O.flash_chunk(d)
    g = O.gpw(d)
    return sorted({2, g, g + 1, k, k + 1, k + 2, 2 * k + 2, 129})


@pytest.mark.parametrize("d", DS)
@pytest.mark.parametrize("regime", O.REGIMES)
def test_flash_emulation_inside_bounds(d, regime):
    """the flash kernel's float32 arithmetic, with perturbed exp / divide / log, stays inside the flash route's bounds"""
    for C in _c_edges(d)[::2] + [_c_edges(d)[-1]]:
        U, T, ids = _case(regime, 16, C, d)
        Q, R = _rows(U, T, ids)
        for mode in (None, "up", "down", "rand"):
            pred, g, row_loss, dq = O.emulate_flash(Q, R, O.Perturb(mode, seed=C))
            ref, _ = O.score_ref(U, None, T, ids)
            assert np.array_equal(pred.astype(np.float64), ref.numpy()), (C, mode)       # Tier A: exact
            L = O.loss_ref(torch.from_numpy(pred), "flash", d)
            for what, msg in (("loss", O.loss_violation(torch.from_numpy(row_loss), L)),
                              ("g", O.g_violation(torch.from_numpy(g), L))):
                assert msg is None, (C, mode, what, msg)
            dqr = O.dq_ref(L.g_in, T, ids)
            msg = O.dq_violation(torch.from_numpy(dq), dqr, O.dq_bound_flash(L, T, ids, d), L)
            assert msg is None, (C, mode, msg)
            assert O.ambiguity_ok(L, regime) is None, (C, O.ambiguity_ok(L, regime))


@pytest.mark.parametrize("regime", O.REGIMES)
def test_loss_kernel_emulation_inside_bounds(regime):
    """k_bpr_loss_rows' float32 arithmetic (expf / logf perturbed) inside the loss route's bounds, and
    rowdot_bwd_query's accumulation of its g inside the separate route's dQ bound"""
    for C in (2, 7, 33, 65, 100):
        U, T, ids = _case(regime, 24, C, 64)
        Q, R = _rows(U, T, ids)
        pred = O.score_ref(U, None, T, ids)[0].float()
        for mode in (None, "up", "down", "rand"):
            g, row_loss = O.emulate_loss(pred.numpy(), O.Perturb(mode, seed=C))
            L = O.loss_ref(pred, "loss")
            assert O.loss_violation(torch.from_numpy(row_loss), L) is None, (C, mode)
            assert O.g_violation(torch.from_numpy(g), L) is None, (C, mode, O.g_violation(torch.from_numpy(g), L))
            dq = O.emulate_bwd_query(g, R)
            msg = O.dq_violation(torch.from_numpy(dq), O.dq_ref(L.g_in, T, ids), O.dq_bound_sep(L, T, ids, 64), L)
            assert msg is None, (C, mode, msg)


def test_clamp_edges_and_c1():
    """C = 1: row loss -log(1e-8f), g and dQ zero; S below 1e-8: exactly zero gradient; S = 1.0f is inside"""
    for d in DS:
        U, T, ids = _case("well", 5, 1, d)
        pred, g, rl, dq = O.emulate_flash(*_rows(U, T, ids))
        assert np.all(g == 0) and np.all(dq == 0)
        assert np.all(rl == np.float32(-math.log(np.float32(1e-8))))
        L = O.loss_ref(torch.from_numpy(pred), "flash", d)
        assert O.loss_violation(torch.from_numpy(rl), L) is None
    U, T, ids = _case("below", 16, 17, 64)
    pred, g, rl, dq = O.emulate_flash(*_rows(U, T, ids))
    L = O.loss_ref(torch.from_numpy(pred), "flash", 64)
    assert not bool(L.inside.any()) and not bool(L.ambiguous.any())
    assert np.all(g == 0) and np.all(dq == 0)
    U, T, ids = _case("straddle", 64, 9, 32)
    L = O.loss_ref(O.score_ref(U, None, T, ids)[0].float(), "flash", 32)
    assert 0 < int(L.inside.sum()) < 64                          # the case sits on the lower edge
    assert np.float32(1.0) - np.float32(1e-8) == np.float32(1.0)  # the upper edge is 1.0f itself


TIGHT = {"flash": 2e-5, "loss": 1e-5}     # the flash route pays __expf / __fdividef (2 ulp each) and its rescales


def test_bounds_are_tight_when_well_conditioned():
    """margins and score spreads <= 4: wherever g_c is not itself cancellation-sized (|s_c^2 - S| >= (s_c + S +
    s_c (1 - s_c)) / 4), the g bound is at most 1e-5 |g_c| on the loss route and 2e-5 |g_c| on the flash route (so is the
    g0 bound); the dQ bound is at most that fraction of the sum of |terms| dQ adds, and at most 2.5x / 5x that of the
    row's norm (dQ's terms cancel: sum_c g_c = 0)"""
    g = torch.Generator().manual_seed(3)
    for d in DS:
        for C in (9, 33, 65):
            tgt = O.quantise(-2 + 4 * torch.rand(64, C, generator=g, dtype=torch.float64))
            U, T, ids = O.exact_operands(tgt, d, g)
            pred = O.score_ref(U, None, T, ids)[0].float()
            for route in O.ROUTES:
                L = O.loss_ref(pred, route, d)
                bar = TIGHT[route]
                assert bool(L.inside.all()) and not bool(L.ambiguous.any())
                br = (L.s * L.s - L.S.unsqueeze(1)).abs()
                keep = br >= (L.s + L.S.unsqueeze(1) + L.s * L.sbar) / 4
                assert int(keep.sum()) > 0.2 * keep.numel()
                rel = L.err_g[:, 1:][keep] / L.g_in[:, 1:].abs()[keep]
                assert float(rel.max()) <= bar, (d, C, route, float(rel.max()))
                assert float((L.err_g0 / L.g_in[:, 0].abs()).max()) <= bar, (d, C, route)
                dqr = O.dq_ref(L.g_in, T, ids)
                bnd = O.dq_bound_flash(L, T, ids, d) if route == "flash" else O.dq_bound_sep(L, T, ids, d)
                assert float((bnd / O.dq_scale(L, T, ids)).max()) <= bar, (d, C, route)
                ratio = float((bnd.norm(dim=1) / dqr.norm(dim=1)).max())
                assert ratio <= (5 if route == "flash" else 2.5) * bar, (d, C, route, ratio)


# ------------------------------------------------------------------------------------------------------------------
# the wrong references
# ------------------------------------------------------------------------------------------------------------------

WRONG_CASES = {          # variant -> regimes of the GPU suite it is checked on
    "detached": ("well", "trained", "asc", "dup"),
    "pos_in_softmax": ("well", "trained", "desc", "dup"),
    "no_clamp": ("below", "huge"),
    "mean_bc": ("well", "trained", "spike", "dup"),
    "sig_flipped": ("well", "trained", "asc", "desc", "dup"),
}


@pytest.mark.parametrize("variant", sorted(WRONG_CASES))
@pytest.mark.parametrize("route", O.ROUTES)
def test_wrong_loss_references_fail_by_10x(variant, route):
    for d in DS:
        for regime in WRONG_CASES[variant]:
            for C in (O.flash_chunk(d) + 1, 100):
                U, T, ids = _case(regime, 32, C, d)
                pred = O.score_ref(U, None, T, ids)[0].float()
                L = O.loss_ref(pred, route, d)
                r = O.wrong_ratio(O.wrong_g(pred, variant), L, L.err_g)
                assert r >= 10, (variant, d, regime, C, r)


def test_wrong_dq_without_positive_term_fails_by_10x():
    for d in DS:
        for regime in ("well", "trained", "dup"):
            U, T, ids = _case(regime, 32, 33, d)
            pred = O.score_ref(U, None, T, ids)[0].float()
            L = O.loss_ref(pred, "flash", d)
            dqr = O.dq_ref(L.g_in, T, ids)
            bnd = O.dq_bound_flash(L, T, ids, d)
            err = (O.wrong_dq_no_g0r0(L, T, ids) - dqr).abs()
            assert float((err / bnd).max()) >= 10, (d, regime)


def test_wrong_tf32_scores_fail_by_10x():
    g = torch.Generator().manual_seed(5)
    for d in (4, 20, 32, 64, 96, 128, 256):
        Q, T = torch.randn(40, d, generator=g), torch.randn(300, d, generator=g)
        qid, ids = torch.randint(0, 40, (50,), generator=g), torch.randint(0, 300, (50, 9), generator=g)
        ref, Sabs = O.score_ref(Q, qid, T, ids)
        bad = O.tf32_scores(Q, qid, T, ids)
        assert float(((bad - ref).abs() / (O.gamma_dot(d) * Sabs)).max()) >= 10, d
        # and an fp32 evaluation of the same dot sits inside
        assert O.score_violation((Q[qid].unsqueeze(1) * T[ids]).sum(2), ref, Sabs, d) is None


@pytest.mark.parametrize("d", DS)
def test_pair_runs_reference_matches_naive_loop_and_wrong_runs_fail(d):
    lpr = d // 4
    key, rows, coef, nk = O.runs_case(lpr, d, n_out=400)
    assert nk < 400
    g = torch.Generator().manual_seed(d)
    T = torch.randn(50, d, generator=g)
    out0 = torch.randn(400, d, generator=g)
    ref, bnd = O.pair_runs_ref(out0, key, rows, coef, T)
    naive = O.pair_runs_naive(out0, key, rows, coef, T)
    assert bool(((ref - naive).abs() <= bnd + 1e-12).all())
    assert torch.equal(ref[nk:], out0[nk:].double())             # keys without a run keep the caller's bits
    for variant in ("cut", "skip_head"):
        bad, _ = O.pair_runs_ref(out0, key, rows, coef, T, variant=variant, lpr=lpr)
        err = (bad - ref).abs()
        assert float((err / torch.where(bnd > 0, bnd, torch.full_like(bnd, 1e-300))).max()) >= 10, variant
    with pytest.raises(ValueError):
        O.pair_runs(np.array([1, 1, -1, 1]), np.array([0, 0, 0, 0]), 5)
    heads, rid = O.pair_runs(np.array([2, 2, 9, 2, 4, 4]), np.array([0, 1, 1, -1, 0, 0]), 5)
    assert heads.tolist() == [0, 4] and rid.tolist() == [0, 0, -1, -1, 1, 1]


# ------------------------------------------------------------------------------------------------------------------
# fixed-order means, rescale count
# ------------------------------------------------------------------------------------------------------------------

def test_tree_means_reproduce_hand_computed_case():
    f = np.float32
    x = np.array([1.0, 2.0 ** -24, 3.0, 2.0 ** -24, 2.0 ** 24], dtype=f)
    # 4 threads: t0 = 1 + 2^24 (rounds to 2^24), t1 = 2^-24, t2 = 3, t3 = 2^-24; tree: (t0 + t2) + (t1 + t3)
    t0, t1, t2, t3 = f(f(1.0) + f(2.0 ** 24)), f(2.0 ** -24), f(3.0), f(2.0 ** -24)
    want = f(f(f(t0 + t2) + f(t1 + t3)) / f(5))
    assert O.tree_mean_f32(x, 4) == want
    assert O.tree_mean_f32(np.ones(1000, f), 256) == f(1) and O.tree_mean_f32(np.ones(3000, f), 1024) == f(1)
    rng = np.random.default_rng(0)
    y = rng.standard_normal(5000).astype(f)
    assert abs(float(O.tree_mean_f32(y, 256)) - float(y.astype(np.float64).mean())) < 1e-6


def test_flash_rescale_count():
    pred = torch.tensor([[0.0, 1, 2, 3, 4, 5, 6, 7, 8, 9], [0.0, 9, 8, 7, 6, 5, 4, 3, 2, 1]])
    # d = 128: one group, chunks of 4 negatives: ascending grows in all 3 chunks, descending only in the first
    assert O.flash_rescales(pred, 128).tolist() == [3.0, 1.0]
    # d = 32: 4 groups x 4 rows = 16 negatives per chunk: a single chunk
    assert O.flash_rescales(pred, 32).tolist() == [1.0, 1.0]
