"""float64 restatement of the first half of a BPR training step -- candidate scoring, the BPR loss and the query-side
gradient dQ -- and the error model its kernels are checked against; test infrastructure, importable without a GPU.

Kernels covered: ``k_bprmf_flash<D>`` (csrc/bprmf_flash.cu), ``k_rowdot_fwd[_generic]``, ``k_rowdot_bwd_query[_generic]``
and ``k_gather_rows[_generic]`` (csrc/rowdot.cu), ``k_bpr_loss_rows`` + ``k_mean_rows`` (csrc/loss.cu), and the shard
owner's ``k_pairdot_fwd[_generic]``, ``k_pairdot_fwd_p2p`` and ``k_pair_runs_sum`` (csrc/pairdot.cu, pairdot_p2p.cu).

The loss (models/BaseModel.py:182-185 restated in oracle/rechorus_oracle.py): for a row x = pred[b] with positive
p = x_0 and negatives x_c (c >= 1), w = softmax(x_1..), s_c = sigmoid(p - x_c), S = sum_c w_c s_c,
loss = -mean_b log(clamp(S, 1e-8, 1 - 1e-8)), and inside the clamp window, with dS = -1 / (B S), e_c = exp(x_c - max),
Z = sum e_c, A = sum e_c s_c, D = sum e_c s_c (1 - s_c):
    g_0 = dS D / Z,     g_c = dS (e_c / Z) ((s_c - S) - s_c (1 - s_c)) = dS (e_c / Z) (s_c^2 - S),
    dQ  = sum_c g_c r_c = g_0 r_0 + (dS / Z) sum_c e_c (s_c^2 - S) r_c.
In float32 1 - 1e-8 rounds to 1.0f, so the window is [1e-8f, 1.0f], upper edge included, in both kernels (and in torch).

Criteria
--------
* Tier A, exact operands (``exact_operands``): every table entry is a multiple of 2^-3 or 2^-6 and every score's sum of
  |terms| stays below 2^16 quanta, so every product and partial sum is a float32 number and a score must equal float64
  bit for bit in any summation order.
* Tier B, a bound per output element that holds for the kernel's arithmetic in any rounding order: scores within
  gamma_dot Sabs; loss, g and dQ within the bounds of ``loss_ref`` / ``dq_bound_*``, evaluated on the kernel's own
  float32 ``pred`` (the flash kernel scores and evaluates the loss from the same registers, so this separates the two).
* Tier C, an accuracy bar on max |got - ref| / scale (``TIER_C``), set from H100 measurements.

Error model (u = 2^-24, one round-to-nearest; U23 = 2^-23 >= one ulp of a normal float32 relative to its value)
------------------------------------------------------------------------------------------------------------------
Constants come from the CUDA C Programming Guide's tables of maximum ulp errors (single precision, no fast-math; the
build passes none): ``expf`` 2 ulp, ``logf`` 1 ulp, IEEE ``x / y`` correctly rounded (u); ``__expf(x)`` 2 + floor(1.173
|x|) ulp; ``__fdividef(x, y)`` 2 ulp for y in [2^-126, 2^126] (all divisors here: Z in [1, C], S in [1e-8, 1], 1 + E
below 2^126 -- beyond, ``__fdividef`` returns 0 and the exact quotient is below 2^-126, the absolute floor TINY).

e_c.  loss.cu: one ``expf`` of the rounded argument x_c - M (M the row max, exact): alpha_c = 2 U23 + u Delta_c,
  Delta_c = M - x_c (a relative argument error u costs u Delta_c of exp).  Flash: e_c = __expf(x - M_j) in chunk j, then
  every running-max rescale multiplies the lane sums by __expf(M_old - M_new) (one more rounding each) and the group
  combine by sg = __expf(M_g - M_all).  The arguments telescope to Delta_c in total, so with R = (number of chunks in which
  some lane group's max grew, ``flash_rescales``) + 2 factors: alpha_c = U23 (2 R + 1.173 Delta_c) + u (Delta_c + R).  The
  e_c the per-candidate gradient loop recomputes is one __expf: alpha'_c = U23 (2 + 1.173 Delta_c) + u Delta_c.
s_c.  s = 1 / (1 + E), E = exp(x - p) with relative error eps_E (flash: U23 (2 + 1.173 |t|) + u |t|; loss.cu: 2 U23 +
  u |t|, t = x - p rounded once).  A relative error eps_E of E moves 1 + E by (1 - s) eps_E relative; + u for the
  addition, + the division's (flash 2 U23, loss.cu u):  sigma_c = (1 - s_c) eps_E + u + div.  Absolute floor TINY.
Sums.  Z, A, D add nonnegative terms; a term passes through at most n_sum roundings (flash: nch chunk additions per lane,
  then log2(LPR) + log2(GPW) = 5 shuffle levels; loss.cu: ceil((C - 1) / 32) per lane + 5), so each sum is within
  gamma(n_sum) of the sum of its computed terms.  A's term e s is one more rounding (u), D's term fma(e s, 1 - s) two.
S = A / Z.  Perturbing the weights e_c by alpha_c moves S by sum_c w_c alpha_c |s_c - S| (the shared e errors cancel
  to first order); s_c by sigma_c moves it by sum_c w_c s_c sigma_c; the sums' roundings and the division add
  S (2 gamma(n_sum) + div):  errS = 1.02 [sum_c w_c (alpha_c |s_c - S| + s_c (sigma_c + u)) + S (2 gamma + div)] + floors.
kz = dS / Z.  dS = -(1/B) / S and the kernel's S times its Z is its A times (1 + division error), so kz's relative
  error is that of A, eps_A = sum_c e_c s_c (alpha_c + sigma_c + u) / A + gamma(n_sum), plus three divisions and two
  products:  eps_kz = eps_A + 3 div + 2 u.
g_c = kz e'_c br_c with br_c = (s_c - S) - s_c (1 - s_c) evaluated in float32.  |delta br_c| <= 2 |delta s_c| + errS +
  3 u (s_c + S + s_c (1 - s_c)) -- the bound scales with s + S + s (1 - s), not with |br|, which is what keeps it valid
  once the sigmoid saturates and br cancels; then
  |delta g_c| <= 1.02 |kz| e_c (|br_c| (eps_kz + alpha'_c + 3 u) + |delta br_c|).
g_0 = kz D.  |delta D| <= sum e_c [s_c (1 - s_c)(alpha_c + sigma_c + 3 u + gamma) + s_c (sigma_c s_c + TINY)] (1 - s is
  formed from the rounded s: its absolute error is that of s);  |delta g_0| <= 1.02 |kz| (D (eps_kz + 2 u) + |delta D|).
loss = -log(clamp(S)).  clamp is 1-Lipschitz and logf 1 ulp:  |delta loss| <= 1.02 errS / clamp(S) + U23 |loss|.
dQ, flash (acc1 = sum e s^2 r, acc2 = sum e r, dQ = fma(g0, r0, kz fma(-S, acc2, acc1))): per lane each acc term passes
  4 nch fmas and log2(GPW) combine additions (n_acc), so with T_c = e_c |r_c|:
    |delta dQ| <= |delta g0| |r0| + u |g0 r0| + 1.02 |kz| [sum T_c ((s^2 + S)(alpha_c + gamma(n_acc)) + 2 s_c (sigma_c s_c
                  + TINY) + 2 u s_c^2 + errS) + |inner| (eps_kz + 3 u)],   inner = sum e_c (s_c^2 - S) r_c.
dQ, separate route (rowdot_bwd_query of the loss kernel's g): gamma(n_bwd) sum |g_c| |r_c| + sum |delta g_c| |r_c|.
Scores.  dot4 is a multiply and three fmas (4 roundings per term), then a butterfly over LPR = d/4 lanes (log2(LPR)
  additions) -- or, generic, ceil(d / 128) chained dot4 per lane and a 5-level warp sum: gamma_dot(d) below.

Clamp window.  A row whose float64 S lies within errS of 1e-8f or of 1.0f may take either branch; such rows are counted
(``LossRef.ambiguous``) and accept either the in-window values or the clamped ones (g = 0, dQ = 0).

The float32 fixed-order means (``tree_mean_f32``) and the run sums of ``k_pair_runs_sum`` (``pair_runs_ref``) are
restated from the kernels' contracts; ``WRONG`` lists deliberately wrong references the bounds must reject.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from tests.linear_tc_oracle import rn_tf32

u = 2.0 ** -24            # unit roundoff of float32, round to nearest
U23 = 2.0 ** -23          # one ulp of a normal float32, relative to its value (upper)
U64 = 2.0 ** -53
TINY = 2.0 ** -126        # absolute floor: flushed or underflowed exp / quotient results
LO = float(np.float32(1e-8))      # clamp window [LO, HI] as float32 compares it
HI = 1.0                          # float32(1 - 1e-8) == 1.0f
ROUTES = ("flash", "loss")

# Tier C bars on max |got - ref| / scale, scale the sum of |terms| each output adds: Sabs for scores, |kz| e_c (s_c + S +
# s_c (1 - s_c)) for g (|kz| A for g_0), ``dq_scale`` for dQ, sum |coef T| for a pair run.  Worst ratios measured on an
# H100 80GB HBM3 (700 W power limit) with tests/test_gpu_bpr_score_loss.py (g and dQ over its well-conditioned cases,
# scores and runs over all of them): score 1.93e-7, g 2.39e-7, dQ 2.97e-7, pair_runs 3.08e-7.  Each bar is at least 4x.
TIER_C = {"score": 8.0e-7, "g": 1.0e-6, "dq": 1.2e-6, "pair_runs": 1.3e-6}


def gamma(k, uu: float = u):
    """gamma(k) = k u / (1 - k u): relative error of k chained roundings"""
    k = k.to(torch.float64) if isinstance(k, torch.Tensor) else float(k)
    return k * uu / (1.0 - k * uu)


def gpw(d: int) -> int:
    """lane groups per warp of the d = 32 / 64 / 128 kernels (LPR = d / 4 lanes per row)"""
    return 128 // d


def flash_chunk(d: int) -> int:
    """negatives per chunk of k_bprmf_flash: GPW groups x 4 rows"""
    return 4 * gpw(d)


def flash_nch(C: int, d: int) -> int:
    return -(-(C - 1) // flash_chunk(d))


# ------------------------------------------------------------------------------------------------------------------
# scores
# ------------------------------------------------------------------------------------------------------------------

def gamma_dot(d: int) -> float:
    """one score of k_rowdot_fwd / k_pairdot_fwd / k_bprmf_flash (d in {32, 64, 128}): 4 roundings in dot4 and
    log2(d / 4) butterfly additions; generic kernels: ceil(d / 128) chained dot4 (4 + 1 roundings each) and 5 levels"""
    if d in (32, 64, 128):
        n = 4 + int(math.log2(d // 4))
    else:
        n = 5 * (-(-d // 128)) + 5
    return gamma(n) + gamma(d, U64)


def score_ref(Q, qid, T, ids):
    """pred[b, c] = <Q[qid[b]], T[ids[b, c]]> (qid None: row b) and Sabs = sum |q_k r_k|, float64 on T's device;
    ids out of range are clamped to row 0, as the kernels do"""
    dev = T.device
    ids = ids.to(dev).clamp(0) * (ids.to(dev) < T.shape[0])
    Qd = Q.to(dev, torch.float64)
    if qid is not None:
        q = qid.to(dev)
        q = q.clamp(0) * (q < Q.shape[0])
        Qd = Qd[q]
    R = T.to(torch.float64)[ids]
    return torch.einsum("bd,bcd->bc", Qd, R), torch.einsum("bd,bcd->bc", Qd.abs(), R.abs())


def pair_ref(Q, qidx, T, rows):
    """out[e] = <Q[qidx[e]], T[rows[e]]>, 0 where rows[e] < 0, and its Sabs"""
    dev = T.device
    rows, qidx = rows.to(dev), qidx.to(dev)
    live = rows >= 0
    r = torch.where(live & (rows < T.shape[0]), rows, torch.zeros_like(rows))
    q = torch.where(live & (qidx >= 0) & (qidx < Q.shape[0]), qidx, torch.zeros_like(qidx))
    Qd, Td = Q.to(dev, torch.float64)[q], T.to(torch.float64)[r]
    m = live.to(torch.float64)
    return (Qd * Td).sum(1) * m, (Qd.abs() * Td.abs()).sum(1) * m


def score_violation(got, ref, Sabs, d: int) -> Optional[str]:
    return _violation(got, ref, gamma_dot(d) * Sabs, "score")


def tf32_scores(Q, qid, T, ids):
    """WRONG reference 7: the scores with both operands rounded to TF32 (what a tf32 tensor-core dot would give)"""
    Qt = torch.from_numpy(rn_tf32(Q.cpu().numpy())).to(T.device)
    Tt = torch.from_numpy(rn_tf32(T.cpu().numpy())).to(T.device)
    return score_ref(Qt, qid, Tt, ids)[0]


# ------------------------------------------------------------------------------------------------------------------
# Tier A operands: scores built to chosen targets, exact in any order
# ------------------------------------------------------------------------------------------------------------------

QUANT = 2.0 ** -6          # targets and all products are multiples of this


def quantise(x: torch.Tensor) -> torch.Tensor:
    return torch.round(x.to(torch.float64) / QUANT) * QUANT


def exact_operands(target: torch.Tensor, d: int, gen: torch.Generator):
    """(U [B, d], T [B C, d], ids [B, C]) float32 with <U[b], T[ids[b, c]]> == target[b, c] exactly.  U[b] = (1, a) and
    T's rows (t - <a, b>, b) with a, b in {-8 .. 8} / 8: every product is a multiple of 2^-6 of magnitude <= 1, and with
    |target| <= 256 every score's sum of |terms| is below (256 + 2 d) 2^6 < 2^16 quanta, so no float32 partial sum in any
    order rounds.  ids are a random permutation of the rows."""
    target = quantise(target)
    if float(target.abs().max()) > 256:
        raise ValueError("targets beyond 256")
    B, C = target.shape
    a = torch.randint(-8, 9, (B, d - 1), generator=gen).double() / 8
    b = torch.randint(-8, 9, (B, C, d - 1), generator=gen).double() / 8
    U = torch.cat([torch.ones(B, 1, dtype=torch.float64), a], 1)
    first = target - torch.einsum("bk,bck->bc", a, b)
    R = torch.cat([first.unsqueeze(2), b], 2).reshape(B * C, d)
    perm = torch.randperm(B * C, generator=gen)
    T = torch.empty_like(R)
    T[perm] = R
    return U.float(), T.float(), perm.reshape(B, C)


def exact_ok(Q, qid, T, ids) -> Optional[str]:
    """Tier A property: every entry a multiple of 2^-6 (after the products: 2^-3 x 2^-3) and every score's sum of
    |terms| below 2^22 quanta.  None when it holds."""
    for name, t in (("Q", Q), ("T", T)):
        x = t.double() * 8
        if not bool((x == torch.round(x)).all()) and not bool(((t.double() / QUANT) == torch.round(t.double() / QUANT)).all()):
            return f"{name} has entries off the 2^-6 grid"
    _, Sabs = score_ref(Q, qid, T, ids)
    if float(Sabs.max()) >= 2.0 ** 22 * QUANT:
        return "sum of |terms| too large"
    return None


def regime_targets(regime: str, B: int, C: int, gen: torch.Generator) -> torch.Tensor:
    """target scores [B, C] (column 0 the positive) for the score regimes of the GPU suite, float64 on the 2^-6 grid"""
    def U(lo, hi, *shape):
        return lo + (hi - lo) * torch.rand(*shape, generator=gen, dtype=torch.float64)
    x = U(-2, 2, B, C)
    if regime in ("well", "dup") or (regime in ("asc", "desc") and C == 1):
        pass
    elif regime == "trained":                      # positive 5 .. 20 above the negatives' mean
        x[:, 0] = x[:, 1:].mean(1) + U(5, 20, B) if C > 1 else U(5, 20, B)
    elif regime in ("asc", "desc") and C > 1:      # the running max moves in every chunk (asc) or never after the first
        n = torch.linspace(-12, 12, max(C - 1, 1), dtype=torch.float64)[: C - 1]
        n = n.unsqueeze(0) + U(-0.1, 0.1, B, C - 1)
        n, _ = torch.sort(n, dim=1, descending=(regime == "desc"))
        x[:, 1:] = n
        x[:, 0] = n.max(1).values + U(-2, 2, B)
    elif regime == "spike":                        # one negative 100 above the rest: the others' weights underflow
        if C > 1:
            j = torch.randint(1, C, (B,), generator=gen)
            x[torch.arange(B), j] = 100 + U(0, 1, B)
            x[:, 0] = 100 + U(-2, 2, B)
    elif regime == "below":                        # S < 1e-8: clamped, g exactly 0
        x[:, 0] = -40 + U(-1, 1, B)
    elif regime == "straddle":                     # S = sigmoid(p - n0) in e^(+-0.25) x 1e-8
        n0 = U(-2, 2, B)
        x[:, 1:] = n0.unsqueeze(1)
        x[:, 0] = n0 + math.log(LO) + torch.linspace(-0.25, 0.25, B, dtype=torch.float64)
    elif regime == "above":                        # S = 1.0f
        x[:, 0] = 40 + U(0, 5, B)
    elif regime == "huge":                         # |x - p| beyond 88: exp over- and underflows inside the sigmoid
        x = U(-120, 120, B, C)
        if C > 1:
            half = torch.arange(B) % 2 == 0
            x[half, 0] = x[half, 1:].max(1).values + U(-5, 5, int(half.sum()))
    else:
        raise ValueError(regime)
    return quantise(x).clamp(-250, 250)


REGIMES = ("well", "trained", "asc", "desc", "spike", "below", "straddle", "above", "huge", "dup")
WELL_CONDITIONED = ("well", "dup")
UPPER_EDGE = ("trained", "above", "huge")      # margins past ~15 put S within a rounding of 1.0f: either branch
LOWER_EDGE = ("straddle",)                     # built to sit on 1e-8f


def add_duplicates(ids: torch.Tensor, gen: torch.Generator) -> torch.Tensor:
    """copy of ids where every sample repeats its positive among the negatives and one negative twice (C >= 3)"""
    ids = ids.clone()
    B, C = ids.shape
    if C >= 2:
        j = torch.randint(1, C, (B,), generator=gen)
        ids[torch.arange(B), j] = ids[:, 0].clone()
    if C >= 4:
        ids[:, C - 1] = ids[:, 2].clone()
    return ids


# ------------------------------------------------------------------------------------------------------------------
# loss and g on the kernel's own pred
# ------------------------------------------------------------------------------------------------------------------

def flash_rescales(pred: torch.Tensor, d: int) -> torch.Tensor:
    """[B] number of chunks of k_bprmf_flash in which some lane group's running max grew (the __any_sync rescales)"""
    B, C = pred.shape
    G, nch = gpw(d), flash_nch(C, d)
    if nch == 0:
        return torch.zeros(B, dtype=torch.float64, device=pred.device)
    x = torch.full((B, nch * 4 * G), -math.inf, dtype=torch.float64, device=pred.device)
    x[:, : C - 1] = pred[:, 1:].to(torch.float64)
    # negative k (0-based) sits in group k % G, chunk k // (4 G)
    xm = x.reshape(B, nch, 4, G).amax(2)                           # [B, nch, G] chunk max per group
    run = torch.cummax(xm, dim=1).values
    prev = torch.cat([torch.full_like(run[:, :1], -math.inf), run[:, :-1]], 1)
    grew = (xm > prev).any(2)
    return grew.sum(1).to(torch.float64)


@dataclass
class LossRef:
    S: torch.Tensor          # [B] float64
    loss: torch.Tensor       # [B] row loss
    g: torch.Tensor          # [B, C] float64 (the clamped branch: zero rows outside the window)
    g_in: torch.Tensor       # [B, C] the in-window formula for every row
    inside: torch.Tensor     # [B] bool
    ambiguous: torch.Tensor  # [B] bool: S within errS of a clamp edge, either branch accepted
    amb_lo: torch.Tensor     # [B] bool: ... of the lower edge 1e-8f
    errS: torch.Tensor
    err_loss: torch.Tensor
    err_g: torch.Tensor      # [B, C] bound on |g_got - g_in|
    kz: torch.Tensor         # [B] dS / Z of the in-window formula
    e: torch.Tensor          # [B, C - 1] exp(x - max)
    s: torch.Tensor
    sbar: torch.Tensor       # 1 - s, formed without cancellation
    alpha: torch.Tensor      # [B, C - 1] relative error bound of the e inside the sums
    sigma: torch.Tensor      # relative error bound of s
    eps_kz: torch.Tensor     # [B]
    err_g0: torch.Tensor     # [B]
    g_scale: torch.Tensor    # [B, C] Tier C scale of g


def _route_consts(route: str, C: int, d: Optional[int]):
    if route == "flash":
        return dict(div=2 * U23, n_sum=flash_nch(C, d) + 5)
    if route == "loss":
        return dict(div=u, n_sum=-(-(C - 1) // 32) + 5)
    raise ValueError(route)


def loss_ref(pred: torch.Tensor, route: str, d: Optional[int] = None) -> LossRef:
    """S, row loss and g in float64 from float32 ``pred`` [B, C], and their bounds for ``route`` ("flash":
    k_bprmf_flash at width d; "loss": k_bpr_loss_rows)"""
    x = pred.to(torch.float64)
    B, C = x.shape
    dev = x.device
    k = _route_consts(route, max(C, 2), d)
    div, gs = k["div"], gamma(k["n_sum"])
    if C == 1:
        z = torch.zeros(B, dtype=torch.float64, device=dev)
        loss = torch.full((B,), -math.log(LO), dtype=torch.float64, device=dev)
        zg = torch.zeros_like(x)
        return LossRef(z, loss, zg, zg, z > 0, z > 0, z > 0, z, U23 * loss, zg, z, x[:, 1:], x[:, 1:], x[:, 1:], x[:, 1:],
                       x[:, 1:], z, z, zg)
    p, n = x[:, :1], x[:, 1:]
    M = n.max(1, keepdim=True).values
    Delta = M - n
    e = torch.exp(-Delta)
    t = n - p
    s, sbar = torch.sigmoid(-t), torch.sigmoid(t)
    Z = e.sum(1)
    A = (e * s).sum(1)
    D = (e * s * sbar).sum(1)
    S = A / Z
    w = e / Z.unsqueeze(1)
    inside = (S >= LO) & (S <= HI)
    Sc = S.clamp(LO, HI)
    loss = -torch.log(Sc)
    Sg = S.clamp_min(1e-300)
    kz = -1.0 / (B * Sg * Z)
    s2 = s * s
    br = s2 - S.unsqueeze(1)
    g_in = torch.empty_like(x)
    g_in[:, 0] = kz * D
    g_in[:, 1:] = kz.unsqueeze(1) * e * br
    # ---- error model ----
    absT = Delta.abs()
    absTt = t.abs()
    if route == "flash":
        R = (flash_rescales(pred, d) + 2).unsqueeze(1)
        alpha = U23 * (2 * R + 1.173 * absT) + u * (absT + R)
        alpha_g = U23 * (2 + 1.173 * absT) + u * absT
        epsE = U23 * (2 + 1.173 * absTt) + u * absTt
    else:
        alpha = 2 * U23 + u * absT
        alpha_g = alpha + u
        epsE = 2 * U23 + u * absTt
    sigma = sbar * epsE + u + div
    ds = sigma * s + TINY                                          # absolute error of s
    Ag = A.clamp_min(1e-300)
    eps_A = (e * s * (alpha + sigma + u)).sum(1) / Ag + gs + (C * TINY) / Ag
    eps_kz = eps_A + 3 * div + 2 * u
    errS = 1.02 * ((w * (alpha * (s - S.unsqueeze(1)).abs() + s * (sigma + u))).sum(1) + S * (2 * gs + div)) \
        + (w * TINY).sum(1) + C * TINY / Z
    err_loss = 1.02 * errS / Sc + U23 * loss + 1e-15 * loss
    scale = s + S.unsqueeze(1) + s * sbar
    dbr = 2 * ds + errS.unsqueeze(1) + 3 * u * scale
    akz = kz.abs().unsqueeze(1)
    err_g = torch.empty_like(x)
    err_g[:, 1:] = 1.02 * akz * (e * (br.abs() * (eps_kz.unsqueeze(1) + alpha_g + 3 * u) + dbr)
                                 + TINY * (br.abs() + dbr)) + TINY
    errD = (e * (s * sbar * (alpha + sigma + 3 * u + gs) + s * ds)).sum(1) + C * TINY
    err_g0 = 1.02 * kz.abs() * (D * (eps_kz + 2 * u) + errD)
    err_g[:, 0] = err_g0
    g_scale = torch.empty_like(x)
    g_scale[:, 0] = kz.abs() * A
    g_scale[:, 1:] = akz * e * scale
    g = g_in * inside.unsqueeze(1)
    amb_lo = (S - LO).abs() <= errS
    amb = amb_lo | ((S - HI).abs() <= errS)
    return LossRef(S, loss, g, g_in, inside, amb, amb_lo, errS, err_loss, err_g, kz, e, s, sbar, alpha, sigma, eps_kz, err_g0,
                   g_scale)


def _violation(got, ref, bnd, what: str) -> Optional[str]:
    err = (got.to(ref.device, torch.float64) - ref).abs()
    bad = ~(err <= bnd)
    if not bool(bad.any()):
        return None
    i = int(torch.argmax(torch.where(bad, (err - bnd).nan_to_num(math.inf), torch.zeros_like(err)).reshape(-1)))
    return (f"{what}: {int(bad.sum())} element(s) out of bound, worst flat index {i}: |err| "
            f"{float(err.reshape(-1)[i]):.3e} > {float(bnd.reshape(-1)[i]):.3e} (ref {float(ref.reshape(-1)[i]):.6e})")


def loss_violation(row_loss, L: LossRef) -> Optional[str]:
    return _violation(row_loss, L.loss, L.err_loss, "row loss")


def g_violation(g, L: LossRef) -> Optional[str]:
    """g within err_g of the in-window formula on rows inside the window, exactly 0 on rows outside; ambiguous rows
    accept either"""
    g = g.to(L.g.device, torch.float64)
    ok_in = ((g - L.g_in).abs() <= L.err_g).all(1)
    ok_out = (g == 0).all(1)
    want_in = L.inside & ~L.ambiguous
    want_out = ~L.inside & ~L.ambiguous
    bad = (want_in & ~ok_in) | (want_out & ~ok_out) | (L.ambiguous & ~ok_in & ~ok_out)
    if not bool(bad.any()):
        return None
    b = int(torch.nonzero(bad)[0])
    if bool(want_out[b]):
        return f"g: {int(bad.sum())} row(s) bad; row {b} is outside the window (S={float(L.S[b]):.3e}) but g != 0"
    return "g (row %d, S=%.3e): " % (b, float(L.S[b])) + str(_violation(g[b], L.g_in[b], L.err_g[b], "g"))


def dq_ref(g_in: torch.Tensor, T: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    R = T.to(torch.float64)[ids.to(T.device).clamp(0) * (ids.to(T.device) < T.shape[0])]
    return torch.einsum("bc,bcd->bd", g_in.to(R.device, torch.float64), R)


def _rows64(T, ids):
    ids = ids.to(T.device)
    return T.to(torch.float64)[ids.clamp(0) * (ids < T.shape[0])]


def dq_bound_flash(L: LossRef, T: torch.Tensor, ids: torch.Tensor, d: int) -> torch.Tensor:
    """[B, d] bound on |dQ_flash - dQ(g_in)| (module docstring); T float32, ids [B, C]"""
    R = _rows64(T, ids).abs()
    B, C = ids.shape
    if C == 1:
        return torch.zeros(B, d, dtype=torch.float64, device=T.device)
    r0, Rn = R[:, 0], R[:, 1:]
    n_acc = 4 * flash_nch(C, d) + int(math.log2(gpw(d))) + 1
    s, S = L.s, L.S.unsqueeze(1)
    coef = L.e * ((s * s + S) * (L.alpha + gamma(n_acc)) + 2 * s * (L.sigma * s + TINY) + 2 * u * s * s
                  + L.errS.unsqueeze(1)) + TINY
    inner = torch.einsum("bc,bcd->bd", L.e * (s * s - S), _rows64(T, ids)[:, 1:]).abs()
    akz = L.kz.abs().unsqueeze(1)
    g0 = L.g_in[:, :1].abs()
    return (L.err_g0.unsqueeze(1) * r0 + u * g0 * r0
            + 1.02 * akz * (torch.einsum("bc,bcd->bd", coef, Rn) + inner * (L.eps_kz.unsqueeze(1) + 3 * u)))


def n_bwd(C: int, d: int) -> int:
    """roundings one term of k_rowdot_bwd_query[_generic] passes: ceil(nchunk / GPS) 8 fmas per lane group, then
    GPS - 1 additions of the groups' partials (generic: C fmas)"""
    if d not in (32, 64, 128):
        return C
    nchunk = -(-C // 8)
    gpc = 256 // (d // 4)
    gps = min(gpc, 1 << max(0, (nchunk - 1).bit_length()))
    return -(-nchunk // gps) * 8 + gps


def dq_bound_sep(L: LossRef, T: torch.Tensor, ids: torch.Tensor, d: int) -> torch.Tensor:
    """[B, d] bound on |rowdot_bwd_query(g_loss) - dQ(g_in)|: gamma(n_bwd) sum |g| |r| + sum |delta g| |r|"""
    R = _rows64(T, ids).abs()
    B, C = ids.shape
    gabs = L.g_in.abs() + L.err_g
    return gamma(n_bwd(C, d)) * torch.einsum("bc,bcd->bd", gabs, R) + torch.einsum("bc,bcd->bd", L.err_g, R)


def dq_scale(L: LossRef, T, ids) -> torch.Tensor:
    """Tier C scale of dQ: |g0| |r0| + |kz| sum e (s^2 + S) |r|"""
    R = _rows64(T, ids).abs()
    if ids.shape[1] == 1:
        return torch.zeros(ids.shape[0], R.shape[2], dtype=torch.float64, device=R.device)
    w = L.e * (L.s * L.s + L.S.unsqueeze(1)) * L.kz.abs().unsqueeze(1)
    return L.g_in[:, :1].abs() * R[:, 0] + torch.einsum("bc,bcd->bd", w, R[:, 1:])


def dq_violation(dq, ref, bnd, L: LossRef) -> Optional[str]:
    """dQ within bnd of ref; rows outside the window exactly 0; ambiguous rows accept either"""
    dq = dq.to(ref.device, torch.float64)
    ok_in = ((dq - ref).abs() <= bnd).all(1)
    ok_out = (dq == 0).all(1)
    want_in = L.inside & ~L.ambiguous
    want_out = ~L.inside & ~L.ambiguous
    bad = (want_in & ~ok_in) | (want_out & ~ok_out) | (L.ambiguous & ~ok_in & ~ok_out)
    if not bool(bad.any()):
        return None
    b = int(torch.nonzero(bad)[0])
    return "dQ (row %d, S=%.3e): " % (b, float(L.S[b])) + str(_violation(dq[b], ref[b], bnd[b], "dQ"))


def worst_ratio(got, ref, scale, rows: Optional[torch.Tensor] = None) -> float:
    """Tier C: max |got - ref| / scale over the elements with scale > 0 (optionally only rows ``rows``)"""
    err = (got.to(ref.device, torch.float64) - ref).abs()
    if rows is not None:
        err, scale = err[rows], scale[rows]
    pos = scale > 0
    if not bool(pos.any()):
        return 0.0
    r = err[pos] / scale[pos]
    return math.inf if bool(torch.isnan(r).any()) else float(r.max())


# ------------------------------------------------------------------------------------------------------------------
# fixed-order float32 means
# ------------------------------------------------------------------------------------------------------------------

def tree_mean_f32(row_loss, nt: int) -> np.float32:
    """thread t of nt sums rows t, t + nt, ... in order; then red[t] += red[t + o] for o = nt/2 .. 1; then / B.
    nt = 256: k_bprmf_flash's last CTA; nt = 1024: k_mean_rows"""
    x = np.asarray(row_loss, dtype=np.float32).reshape(-1)
    B = x.size
    red = np.zeros(nt, dtype=np.float32)
    for i in range(0, B, nt):
        blk = x[i:i + nt]
        red[:blk.size] = (red[:blk.size] + blk).astype(np.float32)
    o = nt // 2
    while o > 0:
        red[:o] = (red[:o] + red[o:2 * o]).astype(np.float32)
        o //= 2
    return np.float32(red[0] / np.float32(B))


# ------------------------------------------------------------------------------------------------------------------
# k_pair_runs_sum
# ------------------------------------------------------------------------------------------------------------------

def pair_runs(key: np.ndarray, rows: np.ndarray, n_out: int):
    """the runs of k_pair_runs_sum's contract: element e is valid when rows[e] >= 0 and 0 <= key[e] < n_out; a run head
    is a valid element whose predecessor is invalid or has another key, and the run is the head and the valid elements
    with its key that follow it.  Returns (heads, run id per element, -1 outside runs); raises when a key forms two runs
    (shard.py never produces that: the kernel would write the row twice)."""
    key, rows = np.asarray(key, dtype=np.int64), np.asarray(rows, dtype=np.int64)
    valid = (rows >= 0) & (key >= 0) & (key < n_out)
    prev_valid = np.concatenate([[False], valid[:-1]])
    prev_key = np.concatenate([[-1], key[:-1]])
    head = valid & (~prev_valid | (prev_key != key))
    rid = np.cumsum(head) - 1
    rid = np.where(valid, rid, -1)
    heads = np.nonzero(head)[0]
    if np.unique(key[heads]).size != heads.size:
        raise ValueError("a key forms two runs")
    return heads, rid


def pair_runs_ref(out0, key, rows, coef, T, variant: Optional[str] = None, lpr: Optional[int] = None):
    """(expected out float64 [n_out, d], bound [n_out, d]): out0 untouched outside the runs' keys (bound 0 there: the
    kernel must keep the caller's bits), out[key] = sum over the run of coef T[rows] with bound gamma(len) sum |coef T|.
    variant "cut": WRONG 8, runs cut at the first LPR-element block boundary after their head; "skip_head": WRONG 9."""
    key_n, rows_n = key.cpu().numpy().astype(np.int64), rows.cpu().numpy().astype(np.int64)
    heads, rid = pair_runs(key_n, rows_n, out0.shape[0])
    e = np.arange(key_n.size)
    use = rid >= 0
    if variant == "cut":
        use &= (e // lpr) == (heads[np.maximum(rid, 0)] // lpr)
    if variant == "skip_head":
        use &= e != heads[np.maximum(rid, 0)]
    dev = T.device
    out = out0.to(dev, torch.float64).clone()
    n_runs = heads.size
    r = torch.from_numpy(np.where(rows_n < T.shape[0], rows_n, 0)[use]).to(dev)
    terms = coef.to(dev, torch.float64)[torch.from_numpy(use).to(dev)].unsqueeze(1) * T.to(torch.float64)[r]
    idx = torch.from_numpy(rid[use]).to(dev)
    sums = torch.zeros((n_runs, T.shape[1]), dtype=torch.float64, device=dev).index_add_(0, idx, terms)
    absums = torch.zeros_like(sums).index_add_(0, idx, terms.abs())
    lens = torch.from_numpy(np.bincount(rid[rid >= 0], minlength=n_runs)).to(dev)
    keys = torch.from_numpy(key_n[heads]).to(dev)
    out[keys] = sums
    bnd = torch.zeros_like(out)
    bnd[keys] = gamma(lens.clamp_min(1)).unsqueeze(1) * absums
    return out, bnd


def runs_case(lpr: int, seed: int, n_out: int = 400, n_min: int = 0):
    """(key, rows, coef, n_keys_used): runs of length 1, LPR - 1, LPR, LPR + 1 and 3 LPR + 5 starting at every offset
    inside an LPR-element block, invalid slots between them (rows < 0, keys < 0 or >= n_out, and -- once -- a valid
    slot of an already used key cut off by an invalid one is avoided: each key forms one run), n not a multiple of LPR;
    repeated with random lengths until n >= n_min.  Keys are 0, 1, 2, ... in order of appearance."""
    rng = np.random.default_rng(seed)
    keys, rows = [], []
    k = 0
    lens = [1, lpr - 1, lpr, lpr + 1, 3 * lpr + 5]

    def filler():
        kind = int(rng.integers(0, 3))
        keys.append([-1, n_out + 3, -7][kind])
        rows.append(int(rng.integers(0, 50)) if kind < 2 else -1)

    for off in range(lpr):
        for ln in lens:
            while len(keys) % lpr != off:
                filler()
            filler()
            while len(keys) % lpr != off:
                filler()
            keys += [k] * ln
            rows += list(rng.integers(0, 50, ln))
            k += 1
    while len(keys) < n_min and k < n_out:
        for _ in range(int(rng.integers(0, 3))):
            filler()
        if not keys or keys[-1] >= 0:
            filler()
        ln = int(rng.integers(1, 3 * lpr + 6))
        keys += [k] * ln
        rows += list(rng.integers(0, 50, ln))
        k += 1
    keys += [-5, 7]                                            # trailing invalid elements, n % LPR != 0
    rows += [3, -1]
    if len(keys) % lpr == 0:
        keys.append(-1)
        rows.append(0)
    if k > n_out:
        raise ValueError("n_out too small")
    n = len(keys)
    return (torch.tensor(keys, dtype=torch.int64), torch.tensor(rows, dtype=torch.int64),
            torch.from_numpy(rng.standard_normal(n).astype(np.float32)), k)


def pair_runs_naive(out0, key, rows, coef, T):
    """per-key loop: out[k] = sum of coef T[rows] over every valid element with key k (equal to the run sum when each
    key forms one run)"""
    out = out0.double().clone()
    touched = set()
    for e in range(key.numel()):
        k, r = int(key[e]), int(rows[e])
        if r < 0 or k < 0 or k >= out.shape[0]:
            continue
        if k not in touched:
            out[k] = 0
            touched.add(k)
        out[k] += float(coef[e]) * T[r if r < T.shape[0] else 0].double()
    return out


# ------------------------------------------------------------------------------------------------------------------
# deliberately wrong references (each must violate the bounds on the suite's cases)
# ------------------------------------------------------------------------------------------------------------------

WRONG = {
    "detached": "softmax weights detached",
    "pos_in_softmax": "the positive included in the softmax",
    "no_clamp": "clamp ignored: rows outside the window keep a gradient",
    "mean_bc": "mean over B C instead of B",
    "sig_flipped": "sigmoid(n - p) instead of sigmoid(p - n)",
    "no_g0r0": "dQ without the positive's g0 r0 term",
    "tf32": "scores computed in TF32",
    "cut": "pair runs cut at the LPR block boundary",
    "skip_head": "run walk skips its head element",
}
LOSS_WRONG = ("detached", "pos_in_softmax", "no_clamp", "mean_bc", "sig_flipped")


def wrong_g(pred, variant: str) -> torch.Tensor:
    """float64 d loss / d pred of a wrong loss formula (LOSS_WRONG), by autograd"""
    x = pred.detach().to(torch.float64).clone().requires_grad_(True)
    B, C = x.shape
    with torch.enable_grad():
        p, n = x[:, :1], x[:, 1:]
        if variant == "pos_in_softmax":
            S = (torch.softmax(x, 1) * torch.sigmoid(p - x)).sum(1)
        else:
            w = torch.softmax(n, 1)
            if variant == "detached":
                w = w.detach()
            s = torch.sigmoid(n - p) if variant == "sig_flipped" else torch.sigmoid(p - n)
            S = (w * s).sum(1)
        ll = -torch.log(S) if variant == "no_clamp" else -torch.log(S.clamp(LO, HI))
        loss = ll.sum() / (B * C) if variant == "mean_bc" else ll.mean()
        loss.backward()
    return x.grad.detach()


def wrong_ratio(got, L: LossRef, bnd: torch.Tensor) -> float:
    """max over the rows that are not ambiguous of |got - the correct clamped value| / bound (inf where the bound is 0
    and got differs): how far a wrong reference sits outside the bound"""
    rows = ~L.ambiguous
    err = (got.to(L.g.device, torch.float64) - L.g).abs()[rows]
    b = bnd[rows]
    if err.numel() == 0:
        return 0.0
    r = torch.where(b > 0, err / b, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max())


def wrong_dq_no_g0r0(L: LossRef, T, ids) -> torch.Tensor:
    g = L.g.clone()
    g[:, 0] = 0
    return dq_ref(g, T, ids)


# ------------------------------------------------------------------------------------------------------------------
# float32 emulations of the kernels' arithmetic (CPU tests of the bounds themselves)
# ------------------------------------------------------------------------------------------------------------------

f32 = np.float32


def _fma(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


class Perturb:
    """moves each exp / divide / log result to the edge of its documented error: mode "up", "down" or "rand" (a seeded
    sign per element)"""

    def __init__(self, mode: Optional[str], seed: int = 0):
        self.mode = mode
        self.rng = np.random.default_rng(seed)

    def __call__(self, r: np.ndarray, ulps) -> np.ndarray:
        r = np.asarray(r, dtype=f32)
        if self.mode is None:
            return r
        if self.mode == "up":
            sgn = np.ones(r.shape, f32)
        elif self.mode == "down":
            sgn = -np.ones(r.shape, f32)
        else:
            sgn = self.rng.choice(np.array([-1, 1], f32), size=r.shape)
        sp = np.spacing(np.abs(r)).astype(f32)
        out = (r.astype(np.float64) + sgn * np.floor(ulps) * sp.astype(np.float64)).astype(f32)
        return np.where(np.isfinite(r) & (r != 0), out, r).astype(f32)


def _expf_fast(y, pert: Perturb):
    y = np.asarray(y, f32)
    with np.errstate(over="ignore", under="ignore"):
        r = np.exp(y.astype(np.float64)).astype(f32)
    r = np.where(r < f32(2.0 ** -126), f32(0), r).astype(f32)         # ex2.approx.ftz flushes denormals
    return pert(r, 2 + np.floor(1.173 * np.abs(y.astype(np.float64))))


def _fdiv_fast(a, b, pert: Perturb):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        r = (a / b).astype(f32)
    r = np.where(np.abs(b) > f32(2.0 ** 126), f32(0), r).astype(f32)
    return pert(r, 2)


def _expf_acc(y, pert: Perturb):
    with np.errstate(over="ignore", under="ignore"):
        r = np.exp(np.asarray(y, np.float64)).astype(f32)
    return pert(r, 2)


def _logf(y, pert: Perturb):
    return pert(np.log(np.asarray(y, np.float64)).astype(f32), 1)


def _butterfly(v: np.ndarray, axis_len: int, ascending: bool = False) -> np.ndarray:
    """v[..., L] float32 lane values -> the butterfly sum every lane ends with (xor distances L/2 .. 1, or 1 .. L/2 for
    the flash kernel's group combine)"""
    os_ = [1 << i for i in range(int(math.log2(axis_len)))]
    for o in (os_ if ascending else os_[::-1]):
        idx = np.arange(axis_len) ^ o
        v = (v + v[..., idx]).astype(f32)
    return v[..., 0]


def _dot_lanes(q: np.ndarray, r: np.ndarray) -> np.ndarray:
    """dot4 per lane: fma(q.x, r.x, fma(q.y, r.y, fma(q.z, r.z, q.w r.w))); q, r [..., LPR, 4]"""
    acc = (q[..., 3] * r[..., 3]).astype(f32)
    for i in (2, 1, 0):
        acc = _fma(q[..., i], r[..., i], acc)
    return acc


def emulate_flash(Q: np.ndarray, R: np.ndarray, pert: Optional[Perturb] = None):
    """k_bprmf_flash's arithmetic in float32 for query rows Q [B, d] and candidate rows R [B, C, d] (column 0 the
    positive): (pred [B, C], g [B, C], row_loss [B], dQ [B, d]).  d/4 lanes per row, 128/d groups taking negatives
    c = 1 + grp + GPW (4 j + k) in chunks of 4, the __any_sync rescale, the group combine with the sg scale, and the
    final g and dQ formulas; every __expf / __fdividef / logf result goes through ``pert``."""
    pert = pert or Perturb(None)
    Q, R = np.asarray(Q, f32), np.asarray(R, f32)
    B, C, d = R.shape
    LPR, G = d // 4, gpw(d)
    RS = LPR // 4
    nch = flash_nch(C, d)
    q = Q.reshape(B, LPR, 4)

    def score(rows):                                  # rows [..., d] -> butterfly over lanes
        return _butterfly(_dot_lanes(q.reshape((B,) + (1,) * (rows.ndim - 2) + (LPR, 4)),
                                     rows.reshape(rows.shape[:-1] + (LPR, 4))), LPR)

    p = score(R[:, 0])
    pred = np.zeros((B, C), f32)
    pred[:, 0] = p
    M = np.full((B, G), -np.inf, f32)
    Zl = np.zeros((B, G, LPR), f32)
    Al = np.zeros((B, G, LPR), f32)
    Dl = np.zeros((B, G, LPR), f32)
    acc1 = np.zeros((B, G, d), f32)
    acc2 = np.zeros((B, G, d), f32)
    for j in range(nch):
        c = 1 + np.arange(G)[:, None] + G * (j * 4 + np.arange(4)[None, :])       # [G, 4]
        valid = c < C
        cc = np.where(valid, c, 0)
        rows = np.where(valid[None, :, :, None], R[:, cc], f32(0))                 # [B, G, 4, d]
        x = score(rows)                                                            # [B, G, 4]
        for gi in range(G):
            for k in range(4):
                if valid[gi, k]:
                    pred[:, c[gi, k]] = x[:, gi, k]
        mx = np.where(valid[None], x, -np.inf).max(2)                              # [B, G]
        trig = (mx > M).any(1)                                                     # [B]
        Mn = np.maximum(M, mx)
        with np.errstate(invalid="ignore"):
            arg = np.where(M == -np.inf, f32(0), (M - Mn).astype(f32))
        sc = np.where(M == -np.inf, f32(1), _expf_fast(arg, pert))
        sc = np.where(trig[:, None], sc, f32(1)).astype(f32)
        M = np.where(trig[:, None], Mn, M).astype(f32)
        Zl = (Zl * sc[:, :, None]).astype(f32)
        Al = (Al * sc[:, :, None]).astype(f32)
        Dl = (Dl * sc[:, :, None]).astype(f32)
        acc1 = (acc1 * sc[:, :, None]).astype(f32)
        acc2 = (acc2 * sc[:, :, None]).astype(f32)
        arg = np.where(valid[None], (x - M[:, :, None]).astype(f32), f32(0))
        e = np.where(valid[None], _expf_fast(arg, pert), f32(0)).astype(f32)
        s = _fdiv_fast(f32(1), (f32(1) + _expf_fast((x - p[:, None, None]).astype(f32), pert)).astype(f32), pert)
        es = (e * s).astype(f32)
        lane = np.arange(4) * RS
        Zl[:, :, lane] = (Zl[:, :, lane] + e).astype(f32)
        Al[:, :, lane] = (Al[:, :, lane] + es).astype(f32)
        Dl[:, :, lane] = _fma(es, (f32(1) - s).astype(f32), Dl[:, :, lane])
        ess = (es * s).astype(f32)
        for k in range(4):
            acc2 = _fma(e[:, :, k, None], rows[:, :, k], acc2)
            acc1 = _fma(ess[:, :, k, None], rows[:, :, k], acc1)
    Z, A, Dp = _butterfly(Zl, LPR), _butterfly(Al, LPR), _butterfly(Dl, LPR)       # [B, G]
    if G > 1:
        Mall = M.max(1, keepdims=True)
        with np.errstate(invalid="ignore"):
            arg = np.where(M == -np.inf, f32(0), (M - Mall).astype(f32))
        sg = np.where(M == -np.inf, f32(0), _expf_fast(arg, pert))
        sg = sg.astype(f32)
        Z, A, Dp = (Z * sg).astype(f32), (A * sg).astype(f32), (Dp * sg).astype(f32)
        acc1 = (acc1 * sg[:, :, None]).astype(f32)
        acc2 = (acc2 * sg[:, :, None]).astype(f32)
        Z, A, Dp = _butterfly(Z, G, True), _butterfly(A, G, True), _butterfly(Dp, G, True)
        acc1 = _butterfly(np.moveaxis(acc1, 1, 2), G, True)
        acc2 = _butterfly(np.moveaxis(acc2, 1, 2), G, True)
        M = Mall[:, 0]
    else:
        Z, A, Dp, acc1, acc2, M = Z[:, 0], A[:, 0], Dp[:, 0], acc1[:, 0], acc2[:, 0], M[:, 0]
    invB = f32(f32(1) / f32(B))
    S = _fdiv_fast(A, Z, pert) if C > 1 else np.zeros(B, f32)
    inside = (S >= f32(1e-8)) & (S <= f32(1) - f32(1e-8))
    dS = np.where(inside, -_fdiv_fast(invB, np.where(inside, S, f32(1)), pert), f32(0)).astype(f32)
    invZ = _fdiv_fast(f32(1), Z, pert) if C > 1 else np.zeros(B, f32)
    g0 = ((dS * Dp).astype(f32) * invZ).astype(f32)
    kz = (dS * invZ).astype(f32)
    r0 = R[:, 0]
    inner = _fma(-S[:, None], acc2, acc1)
    dQ = _fma(g0[:, None], r0, (kz[:, None] * inner).astype(f32))
    Scl = np.minimum(np.maximum(S, f32(1e-8)), f32(1) - f32(1e-8)).astype(f32)
    row_loss = (-_logf(Scl, pert)).astype(f32)
    g = np.zeros((B, C), f32)
    g[:, 0] = g0
    if C > 1:
        xn = pred[:, 1:]
        e = _expf_fast((xn - M[:, None]).astype(f32), pert)
        s = _fdiv_fast(f32(1), (f32(1) + _expf_fast((xn - p[:, None]).astype(f32), pert)).astype(f32), pert)
        br = ((s - S[:, None]).astype(f32) - (s * (f32(1) - s).astype(f32)).astype(f32)).astype(f32)
        g[:, 1:] = ((kz[:, None] * e).astype(f32) * br).astype(f32)
    return pred, g, row_loss, dQ


def emulate_loss(pred: np.ndarray, pert: Optional[Perturb] = None):
    """k_bpr_loss_rows' arithmetic in float32 (32 lanes per row, lane sums then a 5-level butterfly): (g, row_loss)"""
    pert = pert or Perturb(None)
    x = np.asarray(pred, f32)
    B, C = x.shape
    g = np.zeros((B, C), f32)
    if C == 1:
        return g, np.full(B, -_logf(np.full(B, f32(1e-8)), pert), f32)
    p = x[:, 0]
    n = x[:, 1:]
    mx = n.max(1)
    W = -(-(C - 1) // 32) * 32
    npad = np.full((B, W), np.nan, f32)
    npad[:, :C - 1] = n
    lanes = npad.reshape(B, -1, 32)                       # [B, trips, 32]: element c - 1 = trip * 32 + lane
    Z = np.zeros((B, 32), f32)
    A = np.zeros((B, 32), f32)
    Dp = np.zeros((B, 32), f32)
    for it in range(lanes.shape[1]):
        v = lanes[:, it]
        ok = ~np.isnan(v)
        vv = np.where(ok, v, f32(0))
        e = _expf_acc((vv - mx[:, None]).astype(f32), pert)
        s = (f32(1) / (f32(1) + _expf_acc(-(p[:, None] - vv).astype(f32), pert)).astype(f32)).astype(f32)
        Z = np.where(ok, (Z + e).astype(f32), Z)
        A = np.where(ok, _fma(e, s, A), A)
        Dp = np.where(ok, _fma((e * s).astype(f32), (f32(1) - s).astype(f32), Dp), Dp)
    Z, A, Dp = _butterfly(Z, 32), _butterfly(A, 32), _butterfly(Dp, 32)
    S = (A / Z).astype(f32)
    inside = (S >= f32(1e-8)) & (S <= f32(1) - f32(1e-8))
    Sc = np.minimum(np.maximum(S, f32(1e-8)), f32(1) - f32(1e-8)).astype(f32)
    row_loss = (-_logf(Sc, pert)).astype(f32)
    dS = np.where(inside, -(f32(1) / (f32(B) * S).astype(f32)).astype(f32), f32(0)).astype(f32)
    invZ = (f32(1) / Z).astype(f32)
    g[:, 0] = ((dS * Dp).astype(f32) * invZ).astype(f32)
    e = _expf_acc((n - mx[:, None]).astype(f32), pert)
    w = (e * invZ[:, None]).astype(f32)
    s = (f32(1) / (f32(1) + _expf_acc(-(p[:, None] - n).astype(f32), pert)).astype(f32)).astype(f32)
    br = ((s - S[:, None]).astype(f32) - (s * (f32(1) - s).astype(f32)).astype(f32)).astype(f32)
    g[:, 1:] = ((dS[:, None] * w).astype(f32) * br).astype(f32)
    return g, row_loss


def emulate_bwd_query(g: np.ndarray, R: np.ndarray) -> np.ndarray:
    """dQ = sum_c g_c r_c in float32, one fma chain per component (the generic kernel's order)"""
    g, R = np.asarray(g, f32), np.asarray(R, f32)
    acc = np.zeros((R.shape[0], R.shape[2]), f32)
    for c in range(R.shape[1]):
        acc = _fma(g[:, c, None], R[:, c], acc)
    return acc


def ambiguity_ok(L: LossRef, regime: str) -> Optional[str]:
    """rows on a clamp edge are rare outside the regimes built to reach one: at most one per case"""
    n_lo, n_all = int(L.amb_lo.sum()), int(L.ambiguous.sum())
    if regime not in LOWER_EDGE and n_lo > 1:
        return f"{n_lo} rows on the lower clamp edge"
    if regime not in LOWER_EDGE + UPPER_EDGE and n_all > 1:
        return f"{n_all} rows on a clamp edge"
    return None
