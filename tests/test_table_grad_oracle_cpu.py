"""CPU: tests/table_grad_oracle.py against a plain Python loop over positions, on small cases that use every feature of
the contribution contract (two sources, coef, src_id, div, a column-offset source read with ld = 2d, the padding
prefix, ids clamped to row 0, zero coefficients), and its optimizer updates against scalar formulas."""
import math

import numpy as np
import pytest
import torch

from tests import table_grad_oracle as TG


def _loop(ids, n_rows, d, streams, ignore_id, ignore_n):
    """dict row -> [grad (d floats), absum (d floats), count], and the number of clamped ids"""
    out, bad = {}, 0
    flat_of = [s.src.reshape(-1).tolist() for s in streams]
    p = 0
    for si, s in enumerate(streams):
        for q in range(s.n):
            i = int(ids[p])
            if p < ignore_n and i == ignore_id:
                p += 1
                continue
            if i < 0 or i >= n_rows:
                bad += 1
                i = 0
            r = q // s.div
            if s.src_id is not None:
                r = int(s.src_id[r])
            c = 1.0 if s.coef is None else float(s.coef[q])
            e = out.setdefault(i, [[0.0] * d, [0.0] * d, 0])
            for k in range(d):
                x = c * flat_of[si][s.offset + r * s.ld + k]
                e[0][k] += x
                e[1][k] += abs(x)
            e[2] += 1
            p += 1
    return out, bad


def _case(seed, d):
    g = torch.Generator().manual_seed(seed)
    n_rows = 23
    # source 0: the rows of a [12, 2d] buffer read from column d (ld = 2d), div 3, coef, padding prefix
    n0, div0 = 30, 3
    buf = torch.randn(12, 2 * d, generator=g)
    coef0 = torch.randn(n0, generator=g)
    coef0[[4, 17]] = 0.0                                      # zero coefficients still touch their rows
    s0 = TG.Stream(buf, n0, ld=2 * d, offset=d, coef=coef0, src_id=None, div=div0)
    # source 1: src_id into a [7, d] table, div 2, no coef
    n1 = 14
    tab = torch.randn(7, d, generator=g)
    sid = torch.randint(0, 7, ((n1 + 1) // 2,), generator=g)
    s1 = TG.Stream(tab, n1, ld=d, offset=0, coef=None, src_id=sid, div=2)
    ids = torch.randint(0, n_rows, (n0 + n1,), generator=g)
    ids[[0, 5, 9]] = 0                                        # padding inside the prefix ...
    ids[[31, 40]] = 0                                         # ... and the padding id after it, where it counts
    ids[[2, 33]] = n_rows - 1
    ids[[7]] = -4                                             # clamped to row 0 and counted
    ids[[35]] = n_rows + 2
    return ids, n_rows, [s0, s1], 0, n0


@pytest.mark.parametrize("d", [4, 8])
@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_matches_position_loop(seed, d):
    ids, n_rows, streams, ign, ign_n = _case(seed, d)
    ref = TG.table_grad(ids, n_rows, d, streams, ign, ign_n)
    want, bad = _loop(ids, n_rows, d, streams, ign, ign_n)
    assert ref.n_bad == bad == 2
    assert ref.rows.tolist() == sorted(want)
    assert 0 in want and n_rows - 1 in want
    for j, r in enumerate(ref.rows.tolist()):
        gw, aw, kw = want[r]
        assert int(ref.count[j]) == kw
        np.testing.assert_allclose(ref.grad[j].numpy(), gw, rtol=1e-13, atol=1e-13)
        np.testing.assert_allclose(ref.absum[j].numpy(), aw, rtol=1e-13, atol=1e-13)


def test_padding_only_rows_are_untouched_and_ignore_needs_the_prefix():
    d = 4
    src = torch.randn(6, d)
    ids = torch.tensor([0, 0, 3, 0, 0, 0])
    s = TG.Stream(src, 6, ld=d)
    ref = TG.table_grad(ids, 5, d, [s], ignore_id=0, ignore_n=6)
    assert ref.rows.tolist() == [3] and ref.count.tolist() == [1]
    ref = TG.table_grad(ids, 5, d, [s], ignore_id=0, ignore_n=4)              # positions 4, 5 count
    assert ref.rows.tolist() == [0, 3] and ref.count.tolist() == [2, 1]
    assert torch.equal(ref.grad[0], src[4].double() + src[5].double())
    none = TG.table_grad(torch.zeros(3, dtype=torch.int64), 5, d, [TG.Stream(src, 3, ld=d)], 0, 3)
    assert none.rows.numel() == 0 and none.grad.shape == (0, d)


def test_bound_is_gamma_k_plus_one():
    ref = TG.TableGrad(torch.tensor([0]), torch.zeros(1, 2, dtype=torch.float64),
                       torch.tensor([[1.0, 3.0]], dtype=torch.float64), torch.tensor([4]), 0)
    b = ref.bound(torch.tensor([[2.0, -1.0]]))
    g5 = 5 * TG.U / (1 - 5 * TG.U) + 5 * TG.U64 / (1 - 5 * TG.U64)
    assert b.tolist() == [[3.0 * g5, 4.0 * g5]]


def test_optimizer_constants_are_the_kernels_float32_values():
    t = 3
    K = TG.OptConsts.of(1, 1e-3, 0.9, 0.999, 1e-8, 1e-6, 1 - 0.9 ** t, 1 - 0.999 ** t)
    f = np.float32
    assert K.beta1 == float(f(0.9)) and K.omb1 == float(f(1.0 - float(f(0.9))))
    assert K.omb2 == float(f(1.0 - float(f(0.999))))
    assert K.step == float(f(float(f(1e-3)) / float(f(1 - 0.9 ** t))))
    assert K.isb2 == float(f(1.0 / math.sqrt(float(f(1 - 0.999 ** t)))))
    assert K.wd == float(f(1e-6)) and K.eps == float(f(1e-8))
    S = TG.OptConsts.of(0, 0.05, 0.9, 0.999, 0.0, 0.0)
    assert S.step == S.lr == float(f(0.05)) and S.isb2 == 1.0


def test_optimizer_updates_match_scalar_formulas():
    g = torch.Generator().manual_seed(5)
    W0, m0, v0, G = torch.randn(4, 3, generator=g), torch.randn(4, 3, generator=g), torch.rand(4, 3, generator=g), \
        torch.randn(4, 3, generator=g)
    K = TG.OptConsts.of(1, 1e-2, 0.9, 0.999, 1e-8, 1e-3, 0.19, 0.002)
    gg = TG.grad_with_decay(K, G, W0)
    m, v = TG.adam_moments(K, m0, v0, gg)
    W = TG.adam_weight(K, W0, m, v)
    A = TG.OptConsts.of(2, 1e-2, 0.9, 0.999, 1e-10, 0.0)
    va = TG.adagrad_state(A, v0, TG.grad_with_decay(A, G, W0))
    Wa = TG.adagrad_weight(A, W0, va, G.double())
    S = TG.OptConsts.of(0, 1e-2, 0.9, 0.999, 0.0, 1e-3)
    Ws = TG.sgd_weight(S, W0, TG.grad_with_decay(S, G, W0))
    for i in range(4):
        for j in range(3):
            w0, mm, vv, gr = float(W0[i, j]), float(m0[i, j]), float(v0[i, j]), float(G[i, j])
            x = gr + K.wd * w0
            me, ve = K.beta1 * mm + K.omb1 * x, K.beta2 * vv + K.omb2 * x * x
            assert math.isclose(float(m[i, j]), me, rel_tol=1e-15, abs_tol=1e-300)
            assert math.isclose(float(v[i, j]), ve, rel_tol=1e-15, abs_tol=1e-300)
            assert math.isclose(float(W[i, j]), w0 - K.step * me / (math.sqrt(ve) * K.isb2 + K.eps), rel_tol=1e-15)
            vae = vv + gr * gr
            assert math.isclose(float(va[i, j]), vae, rel_tol=1e-15)
            assert math.isclose(float(Wa[i, j]), w0 - A.lr * gr / (math.sqrt(vae) + A.eps), rel_tol=1e-15)
            assert math.isclose(float(Ws[i, j]), w0 - S.lr * (gr + S.wd * w0), rel_tol=1e-15)
