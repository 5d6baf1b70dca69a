"""CPU: the criteria of tests/test_gpu_linear_tc.py checked without a GPU.  Every Tier A case is exactly representable;
the Tier B bound accepts an fp32 emulation of the kernels' split arithmetic summed one term at a time with every
addition rounded toward zero, the Tier C bar the same emulation rounded to nearest, and both reject a single-TF32
(hi*hi only) product, a dropped lo*hi product and a dropped tail row; the grids reach the kernels' edges."""
import numpy as np
import pytest
import torch

from tests import linear_tc_oracle as O

SMS = 132                      # H100 SXM; the boundary-row operands hold for any SM count up to it
FWD, DX, DW = O.fwd_grid(), O.dx_grid(), O.dw_grid()


def test_split_is_hi_plus_lo_to_2_pow_minus_22():
    x = (torch.randn(100000, generator=torch.Generator().manual_seed(0)) * 3).numpy()
    hi, lo = O.split(x)
    assert np.array_equal(O.rn_tf32(hi), hi) and np.array_equal(O.rn_tf32(lo), lo)
    assert not np.array_equal(hi, x)
    assert np.all(np.abs(x.astype(np.float64) - hi - lo) <= 2.0 ** -22 * np.abs(x))
    a = O.with_lo((1000,), torch.Generator().manual_seed(1)).numpy()
    h, l = O.split(a)
    assert np.array_equal(np.abs(h[a != 0]), np.ones(int((a != 0).sum()), dtype=np.float32))
    assert (l != 0).any() and np.array_equal(h.astype(np.float64) + l, a.astype(np.float64))


def test_exact_ok_rejects_what_is_not_exact():
    g = torch.Generator().manual_seed(2)
    assert O.exact_ok(torch.randn(8, 32, generator=g), O.small_ints((4, 32), g)) is not None      # split not exact
    big = O.with_lo((4, 4096), g, zero_frac=0.0)
    assert O.exact_ok(big, torch.ones(2, 4096) * 2) is not None                               # sums past 2^22 quanta
    x, W, b = O.fwd_operands(64, 32, 16, "x", True)
    assert O.exact_ok(x, W, b) is None
    assert O.exact_ok(x, W, b + 2.0 ** -20) is not None                                      # bias off the grid


@pytest.mark.parametrize("i", range(len(FWD)))
def test_forward_tier_a_operands_are_exact(i):
    for lo_in in ("x", "w"):
        x, W, b = O.fwd_case_operands(FWD[i], lo_in)
        assert O.exact_ok(x, W, b) is None, (FWD[i], lo_in)
        hx, lx = O.split(x.numpy())
        hw, lw = O.split(W.numpy())
        # the lo bits sit in the named operand only, so the hi*lo or lo*hi product alone carries them
        assert (lx != 0).any() == (lo_in == "x") and (lw != 0).any() == (lo_in == "w")


@pytest.mark.parametrize("i", range(len(DX)))
def test_dx_tier_a_operands_are_exact(i):
    case = DX[i]
    if case.p == 0.3:
        return                              # float32(W / 0.7) is not exact: Tier B and C only
    s = 2.0 if case.p is not None else 1.0
    for lo_in in ("dy", "w"):
        dy, W, y = O.dx_case_operands(case, lo_in)
        g = dy if y is None else dy * (y > 0).float()
        assert O.exact_ok(g, (W * s).t().contiguous()) is None, (case, lo_in)
        assert (O.split((W * s).numpy())[1] != 0).any() == (lo_in == "w")


@pytest.mark.parametrize("i", range(len(DW)))
def test_dw_tier_a_operands_are_exact(i):
    case = DW[i]
    dy, x, y = O.dw_dense_operands(case.M, case.N, case.K)
    assert O.exact_ok(*O.dw_exact_terms(dy, x, y if case.relu else None)) is None
    for sms in (SMS, 114):
        for lo_in in ("dy", "x"):
            dy, x, y = O.dw_sparse_operands(case.M, case.N, case.K, lo_in, sms)
            A, B = O.dw_exact_terms(dy, x, y if case.relu else None)
            assert O.exact_ok(A, B) is None, (case, lo_in, sms)
            assert (O.split(A.numpy())[1] != 0).any() == (lo_in == "dy")
            assert (O.split(B.numpy())[1] != 0).any() == (lo_in == "x")
            rows = O.dw_boundary_rows(case.M, sms)
            assert case.M - 1 in rows and len(rows) <= 256


@pytest.mark.parametrize("M", [1, 33, 255])
@pytest.mark.parametrize("N,K", [(4, 16), (68, 80), (128, 240)])
def test_dw_small_operands_are_exact(M, N, K):
    for lo_in in ("dy", "x"):
        dy, x, y = O.dw_small_operands(M, N, K, lo_in)
        for yy in (None, y):
            assert O.exact_ok(*O.dw_exact_terms(dy, x, yy)) is None


def test_grids_reach_the_kernel_edges():
    fk = {(c.K, c.N) for c in FWD}
    want = {(K, N) for K in (32, 64, 96, 128) for N in (16, 32, 48, 64, 80, 128, 144, 256) if not (N > 128 and K > 64)}
    assert fk == want
    ms = {c.M for c in FWD}
    assert {4096, 4097, 8191, 200, 204800} <= ms
    assert {c.p for c in FWD} == {None, 0.3, 0.5, 1.0}
    assert {(c.relu, c.bias) for c in FWD} == {(a, b) for a in (False, True) for b in (False, True)}
    # dX: every (N, K) ops.linear_bwd sends to k_linear_tc (linear_tc_shape with K output columns over N)
    dk = {(c.N, c.K) for c in DX}
    assert dk == {(N, K) for N in (32, 64, 96, 128) for K in range(16, 257, 16) if not (K > 128 and N > 64)}
    assert {c.p for c in DX} == {None, 0.5, 0.3} and {c.relu for c in DX} == {False, True}
    wk = {(c.N, c.K) for c in DW}
    assert wk == {(N, K) for N in (4, 8, 60, 64, 68, 124, 128) for K in (16, 32, 48, 64, 80, 240)}
    assert all(c.M % 64 == 1 for c in DW)              # the last CTA's range ends in a one-row slab
    assert {c.p for c in DW} == {None, 0.5, 0.3} and {(c.relu, c.bias) for c in DW} >= {(True, True), (False, False)}


def _fwd_data(M, K, N, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(M, K, generator=g) * 2, torch.randn(N, K, generator=g) * (3 / K ** 0.5), \
        torch.randn(N, generator=g) * 0.5


@pytest.mark.parametrize("M,K,N", [(256, 64, 32), (130, 128, 16), (64, 32, 64)])
def test_forward_criteria_accept_split_arithmetic_and_reject_hi_hi_and_a_dropped_row(M, K, N):
    x, W, b = _fwd_data(M, K, N, M + K + N)
    ref, S = O.fwd_ref(x, W, b, relu=True)
    assert O.bound_violation(O.emulate_fwd(x, W, b, relu=True), ref, S, O.gamma_fwd(K)) is None
    good = O.emulate_fwd(x, W, b, relu=True, rz=False)
    assert O.bound_violation(good, ref, S, O.gamma_fwd(K)) is None
    assert O.ratio(good, ref, S) <= O.TIER_C["fwd"]
    hihi = O.emulate_fwd(x, W, b, relu=True, products=("hh",), rz=False)
    assert O.ratio(hihi, ref, S) > 4 * O.TIER_C["fwd"]
    assert O.bound_violation(hihi, ref, S, O.gamma_fwd(K)) is not None
    no_lohi = O.emulate_fwd(x, W, b, relu=True, products=("hh", "hl"), rz=False)
    assert O.ratio(no_lohi, ref, S) > 4 * O.TIER_C["fwd"]
    tail = good.clone()
    tail[-1] = 0
    assert O.bound_violation(tail, ref, S, O.gamma_fwd(K)) is not None


@pytest.mark.parametrize("M,N,K", [(200, 64, 128), (77, 128, 48)])
def test_dx_criteria_accept_split_arithmetic_and_reject_hi_hi(M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    dy, W = torch.randn(M, N, generator=g) * 0.3, torch.randn(N, K, generator=g) * (3 / N ** 0.5)
    y = torch.randn(M, N, generator=g).clamp_min(0)
    s = np.float32(1 / 0.7)
    ref, S = O.dx_ref(dy, y, W, float(s))
    Wd = (W * torch.tensor(s)).t().contiguous()               # the folded weight, as linear_bwd passes it
    dym = dy * (y > 0).float()
    assert O.bound_violation(O.emulate_fwd(dym, Wd), ref, S, O.gamma_dx(N)) is None
    good = O.emulate_fwd(dym, Wd, rz=False)
    assert O.bound_violation(good, ref, S, O.gamma_dx(N)) is None
    assert O.ratio(good, ref, S) <= O.TIER_C["dx"]
    assert O.ratio(O.emulate_fwd(dym, Wd, products=("hh",), rz=False), ref, S) > 4 * O.TIER_C["dx"]
    unscaled = O.emulate_fwd(dym, W.t().contiguous())         # dropout scale not folded into the weight
    assert O.bound_violation(unscaled, ref, S, O.gamma_dx(N)) is not None
    ge = O.emulate_fwd(dy * (y >= 0).float(), Wd)            # ">=" in the ReLU mask
    assert O.bound_violation(ge, ref, S, O.gamma_dx(N)) is not None


@pytest.mark.parametrize("M,N,K", [(2048, 16, 32), (1000, 8, 48)])
def test_dw_criteria_accept_split_arithmetic_and_reject_hi_hi_and_a_dropped_row(M, N, K):
    g = torch.Generator().manual_seed(M + N + K)
    dy, x = torch.randn(M, N, generator=g) * 0.3, torch.randn(M, K, generator=g) * 2
    rW, SW, rb, Sb = O.dw_ref(dy, None, x)
    rows, _ = O.dw_launch_bounds(M, SMS)
    gamma = O.gamma_dw(M, SMS)
    zW, zb = O.emulate_dw(dy, x, rows)
    assert O.bound_violation(zW, rW, SW, gamma) is None and O.bound_violation(zb, rb, Sb, gamma) is None
    dW, db = O.emulate_dw(dy, x, rows, rz=False)
    assert O.bound_violation(dW, rW, SW, gamma) is None and O.bound_violation(db, rb, Sb, gamma) is None
    assert max(O.ratio(dW, rW, SW), O.ratio(db, rb, Sb)) <= O.TIER_C["dw"]
    hW, hb = O.emulate_dw(dy, x, rows, products=("hh",), rz=False)
    assert O.ratio(hW, rW, SW) > 4 * O.TIER_C["dw"]
    tW, tb = O.emulate_dw(dy[:-1], x[:-1], rows, rz=False)             # the last batch row dropped
    assert O.bound_violation(tW, rW, SW, gamma) is not None and O.bound_violation(tb, rb, Sb, gamma) is not None
    # one CTA's partial dropped from the reduce
    cW, cb = O.emulate_dw(dy[:M - rows // 2], x[:M - rows // 2], rows, rz=False)
    assert O.bound_violation(cW, rW, SW, gamma) is not None
    # dbias left unscaled under dropout: s * sum vs sum
    s = float(np.float32(1 / 0.7))
    _, _, rbs, Sbs = O.dw_ref(dy, None, x, s)
    assert O.bound_violation(db, rbs, Sbs, gamma) is not None


def test_gamma_grows_with_the_reduction():
    assert O.gamma_fwd(32) < O.gamma_fwd(128) < 5e-5
    assert O.dw_launch_bounds(204800, 132) == (1600, 528)
    assert O.dw_launch_bounds(100, 132) == (64, 2)
    assert O.gamma_dw(204800, 132) < 1e-3
