"""GPU: the row-sparse table gradient (index plan: b2r_plan_build_ex + b2r_segment_apply; direct plan:
b2r_direct_plan_build + b2r_direct_plan_apply) and the fused SGD / Adam / Adagrad row update, against the float64
restatement in tests/table_grad_oracle.py.

Part A drives the plans directly over the whole source contract (one or two sources, coef, div, src_id, a column-offset
source read with ld = 2d, the padding prefix, clamped ids) and over the id distributions where the kernels change route
(long rows, spilled buckets, Zipf tails, a single position, nothing but padding).  Part B replays what
RowSparseOptimizer.step() does to every fused table of NeuMF and SASRec at bench size.

Every criterion is a rigorous bound or an exact equality:
  * the summed gradient: |out - ref| <= gamma(k + 1) (A + |dense0|) elementwise, k the row's contributions and A the
    sum of their |coef * src|: true for any summation order, including the cooperative partial sums of long rows;
  * rows the batch does not touch (padding-only rows included) keep their bits; a row with one contribution gets
    exactly float32(dense0 + float32(c * s)); the two plans agree bit for bit on rows with fewer than 48 contributions
    (both sum in ascending position from zero with the same fma); two runs give the same bits;
  * the optimizer: the update's gradient is the mode-1 sum of the same plan (same order, checked by the bound above)
    plus wd * W0, and each of m, v and W is bounded against float64 from the kernel's own inputs, so the summation and
    the update arithmetic are checked apart.
"""
import argparse
import types
from dataclasses import dataclass
from typing import Tuple

import pytest
import torch

from tests import table_grad_oracle as TG

pytestmark = pytest.mark.gpu

U = TG.U
LONG = 48                      # contributions from which the direct plan reduces a row cooperatively (kLong)
LR, BETAS, T = 0.01, (0.9, 0.999), 3


def _dev():
    return torch.device("cuda", 0)


def _within(err, bnd, what):
    bad = ~(err <= bnd)                     # NaN counts as out of bound
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError(f"{what}: {int(bad.sum())} element(s) out of bound, first: |err| "
                             f"{float(err.reshape(-1)[i]):.3e} > {float(bnd.reshape(-1)[i]):.3e}")


def _touched_mask(n_rows, rows):
    t = torch.zeros(n_rows, dtype=torch.bool, device=_dev())
    t[rows] = True
    return t


def _stream(s, d):
    """the oracle's view of an ops.Source: the same storage, offset and leading dimension the kernel is given"""
    return TG.Stream(s.src, s.n, ld=s.ld or d, offset=s.src.storage_offset(), coef=s.coef, src_id=s.src_id, div=s.div)


# ---- shared checks ------------------------------------------------------------------------------------------------

def check_sum(ref, out, dense0, what):
    """touched rows of out (a mode-1 result over dense0, or mode-0 rows when dense0 is None) against the oracle"""
    base = ref.grad if dense0 is None else dense0[ref.rows].double() + ref.grad
    got = out if dense0 is None else out[ref.rows]
    _within((got.double() - base).abs(), ref.bound(None if dense0 is None else dense0[ref.rows]), what)
    one = ref.count == 1                    # exactly one contribution: float32(dense0 + float32(c * s))
    single = ref.grad[one].float()
    want = single if dense0 is None else dense0[ref.rows[one]] + single
    assert torch.equal(got[one], want), f"{what}: single-contribution rows are not exact"


def check_untouched(touched, pairs, what):
    keep = ~touched
    for name, (now, before) in pairs.items():
        if now is not None:
            assert torch.equal(now[keep], before[keep]), f"{what}: untouched rows of {name} changed"


def check_update(K, rows, G, W0, m0, v0, W, m, v, what):
    """the fused update of the touched rows: g = G32 + wd * W0 (G32 = the plan's mode-1 sum); m, v against float64 applied
    to the snapshot and g; W against float64 from W0 and the kernel's own m, v.
      m = fma(b1, m0, fl(omb1 * g32)), g32 = g (1 + d0): |m - m64| <= u b1|m0| + 3.1u omb1|g| <= 4u (b1|m0| + omb1|g|)
      v = fma(b2, v0, fl(fl(omb2 * g32) g32)): the product term carries (1 + u)^4 - 1 < 4.1u, the fma u of the total:
          |v - v64| <= u b2 v0 + 5.1u omb2 g^2 <= 6u (b2 v0 + omb2 g^2)
      Adagrad v = fma(g32, g32, v0): |v - v64| <= u v0 + 3.1u g^2 <= 4u (v0 + g^2)
      W = fma(-step, q, W0), q = m / (sqrt(v) isb2 + eps) to <= ~5e-7 (MUFU rsqrt / divide on the direct plan):
          |W - W64| <= u |W64| + (1 + u) 5e-7 |dW64| <= 4u |W64| + 2e-6 |dW64|
      SGD W = fma(-lr, g32, W0): |W - W64| <= u |W64| + 1.1u lr |g| <= 2u (|W64| + lr |g|)"""
    Wr, W0r = W[rows].double(), W0[rows].double()
    g = TG.grad_with_decay(K, G[rows], W0[rows])
    if K.kind == 0:
        W64 = TG.sgd_weight(K, W0r, g)
        _within((Wr - W64).abs(), 2 * U * (W64.abs() + K.lr * g.abs()), f"{what}: SGD W")
        return
    if K.kind == 1:
        m0r, v0r = m0[rows].double(), v0[rows].double()
        m64, v64 = TG.adam_moments(K, m0r, v0r, g)
        mr, vr = m[rows], v[rows]
        _within((mr.double() - m64).abs(), 4 * U * (K.beta1 * m0r.abs() + K.omb1 * g.abs()), f"{what}: Adam m")
        _within((vr.double() - v64).abs(), 6 * U * (K.beta2 * v0r.abs() + K.omb2 * g * g), f"{what}: Adam v")
        W64 = TG.adam_weight(K, W0r, mr, vr)
    else:
        v0r = v0[rows].double()
        v64 = TG.adagrad_state(K, v0r, g)
        vr = v[rows]
        _within((vr.double() - v64).abs(), 4 * U * (v0r.abs() + g * g), f"{what}: Adagrad state")
        W64 = TG.adagrad_weight(K, W0r, vr, g)
    _within((Wr - W64).abs(), 4 * U * W64.abs() + 2e-6 * (W64 - W0r).abs(), f"{what}: W")


# ---- part A: the kernel contract ------------------------------------------------------------------------------------

@dataclass
class S:
    """one contribution source: n positions, row(p) = p // div (through src_id when set), coef or 1, src rows read from
    column d of a [rows, 2d] buffer with ld = 2d when ld2"""
    n: int
    div: int = 1
    coef: bool = False
    sid: bool = False
    ld2: bool = False


@dataclass
class Case:
    name: str
    plan: str                      # index | direct | both | make (make_plan, asserting which plan it returned)
    d: int
    modes: Tuple[str, ...]         # reduce (mode 0) | dense (mode 1) | sgd | adam | adagrad | adam_clock (mode 2)
    ids: str
    n_rows: int
    src: Tuple[S, ...]
    wd: float = 0.0
    inter: bool = False            # Adam / Adagrad state interleaved per row ([n_rows][2][d], state_ld = 2d)


def _zipf(g, n, n_rows, s=1.2, lo=0):
    k = torch.arange(1, n_rows - lo + 1, dtype=torch.float64)
    cdf = torch.cumsum(k ** -s, 0)
    cdf /= cdf[-1].clone()
    r = torch.searchsorted(cdf, torch.rand(n, generator=g, dtype=torch.float64)).clamp_(max=n_rows - lo - 1)
    return torch.randperm(n_rows - lo, generator=g)[r] + lo


def make_ids(c, g):
    """(ids [n] int64 CPU, ignore_id, ignore_n)"""
    n = sum(s.n for s in c.src)
    n_rows, n0 = c.n_rows, c.src[0].n
    ign, ign_n = -1, 0
    if c.ids == "uniform":
        ids = torch.randint(0, n_rows, (n,), generator=g)
    elif c.ids == "hot":                          # rows just below, at and above the cooperative threshold
        ids = torch.randint(20, n_rows, (n,), generator=g)
        perm = torch.randperm(n, generator=g)
        perm = perm[perm != n // 2]               # (the position that gets row n_rows - 1 below)
        at = 0
        for row, k in ((11, LONG - 1), (12, LONG), (13, LONG + 1), (14, 300)):
            ids[perm[at:at + k]] = row
            at += k
    elif c.ids == "legacy_hot":                   # a hot row, and padding id 0 in the prefix that covers the whole batch
        ids = torch.randint(0, n_rows, (n,), generator=g)
        ids[::3] = 5
        ids[1::7] = 0
        ign, ign_n = 0, n
    elif c.ids == "skew":                         # half the batch in 64 rows: those buckets overflow their regions
        ids = torch.randint(0, n_rows, (n,), generator=g)
        ids[::2] = 1000 + torch.randint(0, 64, ((n + 1) // 2,), generator=g)
    elif c.ids == "zipf":
        ids = _zipf(g, n, n_rows)
        cnt = torch.bincount(ids, minlength=n_rows).sort(descending=True).values
        assert int(cnt[0]) > 65536 and 2048 < int(cnt[1]) <= 65536
    elif c.ids == "zipf_small":
        ids = _zipf(g, n, n_rows)
    elif c.ids == "repeat":                       # NeuMF's user positions with C = div = 100: every row long
        ids = torch.randint(1, n_rows, (n // 100,), generator=g).repeat_interleave(100)
    elif c.ids == "single":
        ids = torch.tensor([n_rows // 3])
    elif c.ids == "allpad":
        ids = torch.zeros(n, dtype=torch.int64)
        ign, ign_n = 0, n
    elif c.ids == "pad":                          # padding id 0 inside the prefix and after it, where it counts
        ids = torch.randint(1, n_rows, (n,), generator=g)
        ids[torch.rand(n, generator=g) < 0.3] = 0
        ign, ign_n = 0, (n0 if len(c.src) == 2 else n // 2)
    elif c.ids == "history":                      # SASRec's item table: Zipf histories right-padded with 0, then scores
        B = n0 // 50
        lengths = torch.randint(1, 51, (B, 1), generator=g)
        hist = _zipf(g, n0, n_rows, lo=1).view(B, 50) * (torch.arange(50).view(1, 50) < lengths)
        ids = torch.cat([hist.reshape(-1), torch.randint(1, n_rows, (n - n0,), generator=g)])
        ign, ign_n = 0, n0
    elif c.ids == "edge":                         # last row, ids out of range (clamped to row 0 and counted)
        ids = torch.randint(0, n_rows, (n,), generator=g)
        ids[::97] = n_rows - 1
        ids[5], ids[50], ids[77] = -3, n_rows, n_rows + 7
    else:
        raise ValueError(c.ids)
    if c.ids not in ("single", "allpad", "legacy_hot", "repeat"):
        ids[n // 2] = n_rows - 1
    return ids, ign, ign_n


def make_sources(c, g):
    from rechorus_b200 import ops
    dev, d, out = _dev(), c.d, []
    for s in c.src:
        nq = (s.n + s.div - 1) // s.div
        R = max(1, nq // 2) if s.sid else nq
        buf = (torch.randn(R, 2 * d if s.ld2 else d, generator=g) * 0.5).to(dev)
        src = buf[:, d:] if s.ld2 else buf
        coef = None
        if s.coef:
            coef = torch.randn(s.n, generator=g)
            coef[7::13] = 0.0                          # zero coefficients still touch their rows
            coef = coef.to(dev)
        sid = torch.randint(0, R, (nq,), generator=g).to(dev) if s.sid else None
        out.append(ops.Source(src=src, n=s.n, coef=coef, src_id=sid, div=s.div, ld=2 * d if s.ld2 else 0))
    return out


K1M = 1_000_000
CASES = [
    # bench shapes: BPRMF's item table (c2), NeuMF's (c3), SASRec's two-stream item table (c4)
    Case("c2_items_direct_adam", "direct", 64, ("adam",), "uniform", K1M, (S(409600, 100, coef=True),), 1e-3, True),
    Case("c2_items_index_srcid", "index", 64, ("dense",), "uniform", K1M, (S(409600, 100, coef=True, sid=True),)),
    Case("c3_mlp_items_ld2d", "make", 64, ("adam",), "uniform", K1M, (S(20480, ld2=True),), 0.0, True),
    Case("c3_users_all_long", "both", 64, ("dense",), "repeat", 50_000, (S(409600, ld2=True),)),
    Case("c3_users_all_long_sgd", "both", 128, ("sgd",), "repeat", 50_000, (S(409600, ld2=True),), 1e-3),
    Case("c4_history_scores_adam", "make", 64, ("adam",), "history", K1M, (S(204800), S(409600, 100, coef=True)),
         1e-3, True),
    Case("c4_history_scores_sgd", "both", 64, ("sgd",), "history", K1M, (S(204800), S(409600, 100, coef=True)), 1e-3),
    Case("c4_history_scores_reduce", "index", 64, ("reduce",), "history", K1M, (S(204800), S(409600, 100, coef=True))),
    # heavy tails: one row above 65,536 and one above 2,048 contributions; skewed buckets that spill
    Case("zipf_dense", "both", 64, ("dense",), "zipf", K1M, (S(614400, 5, coef=True),)),
    Case("zipf_adagrad_direct", "direct", 128, ("adagrad",), "zipf", K1M, (S(614400, 100, coef=True),), 1e-3, True),
    Case("skew_sgd_direct", "direct", 32, ("sgd",), "skew", K1M, (S(20480, 256, coef=True),)),
    Case("skew_adam_index", "index", 32, ("adam",), "skew", K1M, (S(20480, 5, coef=True, sid=True),), 1e-3),
    # rows around the cooperative threshold
    Case("hot_dense", "both", 32, ("dense",), "hot", 1000, (S(5000, 5, coef=True, sid=True),)),
    Case("hot_adam_index_d32", "index", 32, ("adam",), "hot", 1000, (S(5000, coef=True),), 0.0, True),
    Case("hot_adagrad_d20", "index", 20, ("adagrad",), "hot", 1000, (S(5000, coef=True, sid=True),)),
    Case("hot_dense_d4_two_sources", "index", 4, ("dense",), "hot", 1000, (S(2500, 5, coef=True), S(2500, ld2=True))),
    Case("hot_reduce_d256", "index", 256, ("reduce",), "hot", 1000, (S(5000, 100, coef=True),)),
    # padding: nothing but padding; padding id after the prefix, where it counts
    Case("allpad_adam", "both", 64, ("adam", "dense"), "allpad", 50, (S(700),), 1e-3, True),
    Case("allpad_reduce_d4", "index", 4, ("reduce",), "allpad", 50, (S(300),)),
    Case("pad_two_sources_dense", "both", 64, ("dense",), "pad", 40, (S(3000, coef=True), S(3000, 5, coef=True))),
    Case("pad_two_sources_adagrad", "both", 32, ("adagrad",), "pad", 300, (S(3000, ld2=True), S(3000, 5, coef=True)),
         1e-3, True),
    Case("pad_reduce_two_sources", "index", 64, ("reduce",), "pad", 3000, (S(3000), S(3000, 5, coef=True, sid=True))),
    # a single position; ids at n_rows - 1 and out of range
    Case("single_dense", "both", 128, ("dense", "sgd"), "single", 1000, (S(1, coef=True),)),
    Case("single_reduce_d20", "index", 20, ("reduce",), "single", 1000, (S(1),)),
    Case("edge_dense", "both", 32, ("dense",), "edge", 777, (S(5000, 5, coef=True),)),
    Case("edge_adam_d256", "index", 256, ("adam",), "edge", 4000, (S(1500, coef=True, sid=True), S(1500, ld2=True)),
         1e-3, True),
    # generic-d kernels, make_plan's choice, the device clock
    Case("make_d20_sgd", "make", 20, ("sgd",), "uniform", 30000, (S(20000, 100, coef=True, ld2=True),), 1e-3),
    Case("make_d256_adam_clock", "make", 256, ("adam_clock",), "uniform", 100_000, (S(30000, 256, coef=True),), 1e-3),
    Case("direct_d128_adam_clock", "direct", 128, ("adam_clock",), "uniform", 100_000,
         (S(50000, 5, coef=True, sid=True),), 0.0, True),
    Case("d4_adam_two_sources", "index", 4, ("adam",), "zipf_small", 500, (S(10000, 100, coef=True), S(10000)),
         1e-3, True),
    Case("d64_adagrad_index_two_sources", "index", 64, ("adagrad",), "uniform", 20000,
         (S(8000, 5, coef=True), S(8000, ld2=True)), 1e-3, True),
    # the shapes the index and direct plans were first cross-checked on
    Case("legacy_uniform", "both", 64, ("dense", "adam"), "uniform", 1000, (S(5000, coef=True),), 1e-4),
    Case("legacy_7rows_long", "both", 64, ("dense", "adam"), "uniform", 7, (S(2560, coef=True),), 1e-4),
    Case("legacy_3rows_oversize", "both", 64, ("dense", "adam"), "uniform", 3, (S(9000, coef=True),), 1e-4),
    Case("legacy_sparse_d32", "both", 32, ("dense", "adam"), "uniform", 100_000, (S(3000, coef=True),), 1e-4),
    Case("legacy_d128", "both", 128, ("dense", "adam"), "uniform", 50, (S(700, coef=True),), 1e-4),
    Case("legacy_hot_ignore", "both", 64, ("dense", "adam"), "legacy_hot", 40, (S(6000, coef=True),), 1e-4),
]


class _Plans:
    """builds a fresh plan of one kind for the case's ids, checking the out-of-range counter every time"""

    def __init__(self, c, ids, ign, ign_n, n_bad):
        self.c, self.ids, self.ign, self.ign_n, self.n_bad = c, ids, ign, ign_n, n_bad

    def build(self, kind):
        from rechorus_b200 import ops
        flag = ops.err_flag(_dev())
        flag.zero_()
        if kind == "make":
            P = ops.make_plan(self.ids, self.c.n_rows, self.c.d, self.ign, self.ign_n)
            want = ops.DirectPlan if self.c.d in ops.DirectPlan.SUPPORTED_D else ops.IndexPlan
            assert type(P) is want, type(P)
        else:
            P = (ops.IndexPlan if kind == "index" else ops.DirectPlan)(self.ids, self.c.n_rows, self.ign, self.ign_n)
        assert int(flag.item()) == self.n_bad
        if self.n_bad:
            with pytest.raises(IndexError):
                ops.check_ids()
        ops.check_ids()
        return P


def _opt(kind, wd, state_ld, clock=None):
    from rechorus_b200 import lib as L
    k = {"sgd": 0, "adam": 1, "adam_clock": 1, "adagrad": 2}[kind]
    eps = {0: 0.0, 1: 1e-8, 2: 1e-10}[k]
    if clock is not None:                      # the bias corrections come from the clock: the host fields are ignored
        return L.Optim(k, LR, BETAS[0], BETAS[1], eps, wd, 0.5, 0.5, state_ld, clock.data_ptr())
    return L.Optim(k, LR, BETAS[0], BETAS[1], eps, wd, 1 - BETAS[0] ** T, 1 - BETAS[1] ** T, state_ld)


def _consts(o):
    return TG.OptConsts.of(o.kind, o.lr, o.beta1, o.beta2, o.eps, o.weight_decay, o.bc1, o.bc2)


def _state(c, gd):
    """W0, m0, v0 (m0 / v0 None where the optimizer has no such state); every fifth row starts from zero state"""
    n_rows, d, dev = c.n_rows, c.d, _dev()
    W0 = torch.randn(n_rows, d, device=dev, generator=gd) * 0.3
    if c.inter:
        mv = torch.empty(n_rows, 2, d, device=dev)
        m0, v0 = mv[:, 0, :], mv[:, 1, :]
    else:
        m0, v0 = torch.empty(n_rows, d, device=dev), torch.empty(n_rows, d, device=dev)
    m0.copy_(torch.randn(n_rows, d, device=dev, generator=gd) * 1e-2)
    v0.copy_(torch.rand(n_rows, d, device=dev, generator=gd) * 1e-4)
    zero = torch.arange(n_rows, device=dev) % 5 == 0
    m0[zero] = 0.0
    v0[zero] = 0.0
    return W0, m0, v0


def _clone_state(c, m0, v0):
    if c.inter:
        mv = torch.stack([m0, v0], 1).contiguous()
        return mv[:, 0, :], mv[:, 1, :]
    return m0.clone(), v0.clone()


def _run_optim(c, kind, mode, P_build, sources, ref, touched, gd):
    from rechorus_b200 import lib as L, ops
    d = c.d
    W0, m0, v0 = _state(c, gd)
    state_ld = 2 * d if c.inter else 0
    # the update's gradient: the same plan's mode-1 sum from zero (same rows, same order)
    G = torch.zeros(c.n_rows, d, device=_dev())
    P_build().add_to_dense(G, sources)
    check_sum(ref, G, torch.zeros_like(G), f"{c.name}/{kind}/{mode} G32")
    assert not bool(G[~touched].any())
    o = _opt(mode, c.wd, state_ld)
    W = W0.clone()
    m, v = _clone_state(c, m0, v0)
    P_build().apply_optimizer(W, m if o.kind == 1 else None, v if o.kind != 0 else None, o, sources)
    check_untouched(touched, {"W": (W, W0), "m": (m, m0), "v": (v, v0)}, f"{c.name}/{kind}/{mode}")
    check_update(_consts(o), ref.rows, G, W0, m0, v0, W, m, v, f"{c.name}/{kind}/{mode}")
    # same bits on a second run
    W2 = W0.clone()
    m2, v2 = _clone_state(c, m0, v0)
    if mode == "adam_clock":                   # ... and with the step constants taken from the device clock
        clock = torch.zeros(4, device=_dev())
        for _ in range(T):
            L.check(L.load().b2r_optim_tick(clock.data_ptr(), LR, BETAS[0], BETAS[1], ops._stream()), "b2r_optim_tick")
        o = _opt(mode, c.wd, state_ld, clock)
    P_build().apply_optimizer(W2, m2 if o.kind == 1 else None, v2 if o.kind != 0 else None, o, sources)
    assert torch.equal(W2, W) and torch.equal(m2, m) and torch.equal(v2, v), f"{c.name}/{kind}/{mode}: not reproducible"
    return W


def _run_dense(c, kind, P_build, sources, ref, touched, gd):
    dense0 = torch.randn(c.n_rows, c.d, device=_dev(), generator=gd) * 0.5
    out = dense0.clone()
    P_build().add_to_dense(out, sources)
    check_untouched(touched, {"dense": (out, dense0)}, f"{c.name}/{kind}/dense")
    check_sum(ref, out, dense0, f"{c.name}/{kind}/dense")
    out2 = dense0.clone()
    P_build().add_to_dense(out2, sources)
    assert torch.equal(out, out2), f"{c.name}/{kind}: not reproducible"
    return out


def _run_reduce(c, P_build, sources, ref):
    P = P_build()
    uniq, rows = P.reduce_rows(c.d, sources)
    assert torch.equal(uniq, ref.rows)
    check_sum(ref, rows, None, f"{c.name}/reduce")
    uniq2, rows2 = P_build().reduce_rows(c.d, sources)
    assert torch.equal(uniq2, uniq) and torch.equal(rows2, rows)


@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_plan_apply_matches_float64(c):
    seed = sum(ord(ch) * (i + 1) for i, ch in enumerate(c.name))
    g = torch.Generator().manual_seed(seed)
    ids, ign, ign_n = make_ids(c, g)
    ids = ids.to(_dev())
    sources = make_sources(c, g)
    ref = TG.table_grad(ids, c.n_rows, c.d, [_stream(s, c.d) for s in sources], ign, ign_n)
    touched = _touched_mask(c.n_rows, ref.rows)
    plans = _Plans(c, ids, ign, ign_n, ref.n_bad)
    kinds = ("index", "direct") if c.plan == "both" else (c.plan,)
    gd = torch.Generator(device=_dev())
    outs = {}
    for mode in c.modes:
        for kind in kinds:
            gd.manual_seed(seed)                # same starting state for both plans
            build = lambda: plans.build(kind)   # noqa: E731
            if mode == "reduce":
                _run_reduce(c, build, sources, ref)
            elif mode == "dense":
                outs[kind, mode] = _run_dense(c, kind, build, sources, ref, touched, gd)
            else:
                outs[kind, mode] = _run_optim(c, kind, mode, build, sources, ref, touched, gd)
        if c.plan == "both" and mode in ("dense", "sgd"):
            # both plans sum a short row in ascending position from zero with the same fma: same bits
            short = ref.rows[ref.count < LONG]
            assert torch.equal(outs["index", mode][short], outs["direct", mode][short])


# ---- part B: the models at bench size --------------------------------------------------------------------------------

def _build(name, extra, n_users, n_items):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = argparse.ArgumentParser()
    p = BaseRunner.parse_runner_args(p)
    p = cls.parse_model_args(p)
    a = p.parse_args(extra + ["--table_mode", "fused"])
    a.device, a.model_path = _dev(), "/tmp/_b2r_unused.pt"
    torch.manual_seed(0)
    m = cls(a, types.SimpleNamespace(n_users=n_users, n_items=n_items)).to(a.device)
    m.train()
    return m


def _neumf_batches(g, B, C, n_users, n_items):
    uid, iid, out = None, None, []
    for _ in range(3):
        u = torch.randint(1, n_users, (B,), generator=g)
        i = torch.randint(1, n_items, (B, C), generator=g)
        if uid is not None:                     # half of the batch reused: some rows skip a step, some do not
            u[: B // 2], i[: B // 2] = uid[: B // 2], iid[: B // 2]
        uid, iid = u, i
        feed = {"user_id": u.to(_dev()), "item_id": i.to(_dev()), "batch_size": B, "phase": "train"}
        out.append((feed, {"mf_u_embeddings": u, "mlp_u_embeddings": u, "mf_i_embeddings": i,
                           "mlp_i_embeddings": i}))
    return out


def _sasrec_batches(g, B, C, L, n_items):
    prev, out = None, []
    for _ in range(3):
        lengths = torch.randint(1, L + 1, (B,), generator=g)
        hist = _zipf(g, B * L, n_items, lo=1).view(B, L) * (torch.arange(L).view(1, L) < lengths.view(B, 1))
        iid = torch.randint(1, n_items, (B, C), generator=g)
        if prev is not None:
            h0, l0, i0 = prev
            hist[: B // 2], lengths[: B // 2], iid[: B // 2] = h0[: B // 2], l0[: B // 2], i0[: B // 2]
        prev = hist, lengths, iid
        feed = {"user_id": torch.zeros(B, dtype=torch.int64, device=_dev()), "item_id": iid.to(_dev()),
                "history_items": hist.to(_dev()), "lengths": lengths.to(_dev()), "batch_size": B, "phase": "train"}
        out.append((feed, {"i_embeddings": torch.cat([hist[hist != 0], iid.reshape(-1)])}))
    return out


def _fused_step_matches_float64(monkeypatch, m, batches, plan_type):
    from rechorus_b200 import ops
    from rechorus_b200.optim import RowSparseOptimizer
    opt = RowSparseOptimizer(m, "Adam", lr=1e-3, l2=1e-6)
    m.optimizer = opt
    tables = {name.split(".")[0]: p for name, p in m.named_parameters() if any(p is t for t in m.sparse_tables())}
    real_make_plan = ops.make_plan
    seen = {}

    def spy_make_plan(ids, n_rows, d, ignore_id=-1, ignore_n=0):
        plan = real_make_plan(ids, n_rows, d, ignore_id, ignore_n)
        assert type(plan) is plan_type, type(plan)
        real_apply = plan.apply_optimizer

        def apply_optimizer(W, mm, vv, o, sources):
            # replayed before the real update: a direct plan of the same (n, n_rows) shares its cached workspace, and the
            # replay rebuilds it from the same ids before the real apply reads it
            G = torch.zeros_like(W)
            type(plan)(ids, n_rows, ignore_id, ignore_n).add_to_dense(G, sources)
            ref = TG.table_grad(ids, n_rows, d, [_stream(s, d) for s in sources], ignore_id, ignore_n)
            assert ref.n_bad == 0
            check_sum(ref, G, torch.zeros_like(G), f"G32 of the table at {W.data_ptr():#x}")
            seen[W.data_ptr()] = (G, ref, _consts(o))
            real_apply(W, mm, vv, o, sources)

        plan.apply_optimizer = apply_optimizer
        return plan

    monkeypatch.setattr(ops, "make_plan", spy_make_plan)
    for step, (feed, used) in enumerate(batches):
        opt.zero_grad()
        m.loss(m(feed)).backward()
        snap = {}
        for name, p in tables.items():
            e = opt.entry(p)
            snap[name] = (p.detach().clone(), e["m"].clone(), e["v"].clone())
        seen.clear()
        opt.step()
        ops.check_ids()
        assert len(seen) == len(tables)
        for name, p in tables.items():
            e = opt.entry(p)
            G, ref, K = seen[p.data_ptr()]
            what = f"step {step} {name}"
            assert torch.equal(ref.rows.cpu(), torch.unique(used[name])), what
            W0, m0, v0 = snap[name]
            touched = _touched_mask(p.shape[0], ref.rows)
            check_untouched(touched, {"W": (p.detach(), W0), "m": (e["m"], m0), "v": (e["v"], v0)}, what)
            check_update(K, ref.rows, G, W0, m0, v0, p.detach(), e["m"], e["v"], what)
            assert K.kind == 1 and K.wd == TG.f32(1e-6) and e["state_ld"] == 2 * p.shape[1]


MODELS = [
    ("neumf_c3", "NeuMF", ["--emb_size", "64", "--layers", "[64, 32, 16]", "--num_neg", "4"], 1_000_000, 1_000_000, 5),
    ("neumf_c100_long_users", "NeuMF", ["--emb_size", "64", "--layers", "[64, 32, 16]", "--num_neg", "99"], 50_000,
     1_000_000, 100),
    ("neumf_d48_index_plan", "NeuMF", ["--emb_size", "48", "--layers", "[64, 32, 16]", "--num_neg", "4"], 200_000,
     200_000, 5),
]


@pytest.mark.parametrize("case", MODELS, ids=[c[0] for c in MODELS])
def test_neumf_fused_adam_steps_match_float64(monkeypatch, case):
    from rechorus_b200 import ops
    _, name, args, n_users, n_items, C = case
    m = _build(name, args, n_users, n_items)
    d = m.emb_size
    batches = _neumf_batches(torch.Generator().manual_seed(C + d), 4096, C, n_users, n_items)
    _fused_step_matches_float64(monkeypatch, m, batches,
                                ops.DirectPlan if d in ops.DirectPlan.SUPPORTED_D else ops.IndexPlan)


def test_sasrec_c4_fused_adam_steps_match_float64(monkeypatch):
    from rechorus_b200 import ops
    n_items, B, C, L = 1_000_000, 4096, 100, 50
    m = _build("SASRec", ["--emb_size", "64", "--history_max", str(L), "--num_layers", "2", "--num_heads", "4",
                          "--num_neg", str(C - 1)], 10, n_items)
    batches = _sasrec_batches(torch.Generator().manual_seed(4), B, C, L, n_items)
    _fused_step_matches_float64(monkeypatch, m, batches, ops.DirectPlan)
