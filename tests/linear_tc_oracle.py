"""float64 restatement of the tensor-core Linear kernels (csrc/linear_tc.cu: forward and masked dX; csrc/linear_dw_tc.cu:
dW and dbias) and the error model they are checked against -- test infrastructure, importable without a GPU.

Three criteria, from strict to loose:
  * Tier A, exact operands: every hi / lo half of the TF32 split, every product the kernel forms and every partial sum
    is an fp32 number, so the kernel must equal float64 bit for bit in any summation order (``exact_ok`` states the
    property, ``fwd_operands``, ``dw_dense_operands`` and ``dw_sparse_operands`` build such cases);
  * Tier B, a bound that holds for any fp32 accumulation order or rounding mode: |got - ref| <= gamma S + c 2^-24 |ref|
    elementwise, S the float64 sum of |terms| (``gamma_fwd``, ``gamma_dx``, ``gamma_dw`` derive gamma);
  * Tier C, an accuracy bar on max |got - ref| / S, set from H100 measurements (``TIER_C``): a single TF32 product
    (hi*hi only) is two to three orders of magnitude above it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import torch

U23 = 2.0 ** -23          # one fp32 addition in any rounding mode (truncation included)
U24 = 2.0 ** -24          # one round-to-nearest fp32 operation
LO_STEP = 2.0 ** -13      # Tier A: the lo half of a split operand is a multiple of this, below TF32 precision of 1

# Tier C bars on max |got - ref| / S.  Worst ratios measured on an H100 80GB HBM3 (700 W power limit) over the whole
# grid and the NeuMF / SASRec replays of tests/test_gpu_linear_tc.py: forward 1.30e-6, dX 1.66e-6, dW 3.12e-7 (NeuMF's
# 16 x 32 layer at 20,480 rows; 1.09e-7 over the grid).  Each bar is at least 4x that.  A hi*hi-only product gives
# 1.5e-4 .. 2.7e-4 on the forward and 3.5e-5 .. 4.8e-5 on dW at the shapes of tests/test_linear_tc_oracle_cpu.py.
TIER_C = {"fwd": 7.0e-6, "dx": 7.0e-6, "dw": 1.3e-6}


# ------------------------------------------------------------------------------------------------------------------
# the TF32 split (tc_rn_tf32 / tc_split in csrc/linear_tc.cuh, dw_rn_tf32 in csrc/linear_dw_tc.cu)
# ------------------------------------------------------------------------------------------------------------------

def rn_tf32(x: np.ndarray) -> np.ndarray:
    """round float32 to 10 explicit mantissa bits, ties away from zero: (bits + 0x1000) & 0xFFFFE000"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def split(x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """hi = rn_tf32(x), lo = rn_tf32(x - hi) (x - hi is exact in fp32)"""
    x = np.asarray(x, dtype=np.float32)
    hi = rn_tf32(x)
    lo = rn_tf32((x - hi).astype(np.float32))
    return hi, lo


# ------------------------------------------------------------------------------------------------------------------
# float64 references: (ref, S) with S the sum of |terms| that ref adds
# ------------------------------------------------------------------------------------------------------------------

def _d(t, device):
    return t.to(device=device, dtype=torch.float64)


def fwd_ref(x, W, bias=None, relu=False, keep=None, s=1.0, device="cpu"):
    """Y = keep * s * act(x W^T + b) and S = keep * s * (|x| |W|^T + |b|), float64 on ``device``"""
    x64, W64 = _d(x, device), _d(W, device)
    z = x64 @ W64.t()
    S = x64.abs() @ W64.abs().t()
    if bias is not None:
        b64 = _d(bias, device)
        z = z + b64
        S = S + b64.abs()
    if relu:
        z = z.clamp_min(0.0)
    if keep is not None:
        k = _d(keep, device) * s
        z, S = z * k, S * k
    return z, S


def dx_ref(dy, y_relu, W, s=1.0, device="cpu"):
    """dX = (dy o [y > 0]) (s W) and S = |dy o [y > 0]| (s |W|); s is the float32 dropout scale the weight is folded with"""
    g = _d(dy, device)
    if y_relu is not None:
        g = g * (_d(y_relu, device) > 0)
    W64 = _d(W, device) * s
    return g @ W64, g.abs() @ W64.abs()


def dw_ref(dy, y_relu, x, s=1.0, device="cpu"):
    """dW = s (dy o [y > 0])^T x, db = s sum_m (dy o [y > 0]) and their S"""
    g = _d(dy, device)
    if y_relu is not None:
        g = g * (_d(y_relu, device) > 0)
    x64 = _d(x, device)
    return (s * (g.t() @ x64), s * (g.abs().t() @ x64.abs()), s * g.sum(0), s * g.abs().sum(0))


# ------------------------------------------------------------------------------------------------------------------
# Tier B: gamma of each kernel
# ------------------------------------------------------------------------------------------------------------------

def split_error(products: int) -> float:
    """Relative error of one product x w formed from TF32 halves.  hi = rn_tf32(x) has |x - hi| <= 2^-11 |x|, lo =
    rn_tf32(x - hi) has |x - hi - lo| <= 2^-11 |x - hi| <= 2^-22 |x| and |lo| <= (2^-11 + 2^-22) |x|; each hi*hi, hi*lo,
    lo*hi, lo*lo is exact in fp32 (11 x 11 significant bits).
      4 products: x w - (hx + lx)(hw + lw) = ex w + (hx + lx) ew        -> <= (2 + 2^-21) 2^-22 |x w| < 3 * 2^-22
      3 products: the same minus lx lw, |lx lw| <= (1 + 2^-11)^2 2^-22  -> <  4 * 2^-22"""
    return {3: 4 * 2.0 ** -22, 4: 3 * 2.0 ** -22}[products]


def gamma_fwd(K: int) -> float:
    """k_linear_tc, one output: 3 K exact products (hi*hi, hi*lo, lo*hi over K) added into one fp32 accumulator, then
    + bias.  Each addition, whatever its order, rounding mode or the tensor core's internal alignment, perturbs the
    running sum by at most 2^-23 of its magnitude, and every running sum is at most S (1 + O(2^-20)): 3 K + 1 additions
    give (3 K + 1) 2^-23 S.  With the split error: gamma = 4 * 2^-22 + (3 K + 1) 2^-23 (x 1.01 for the second-order
    terms).  ReLU is 1-Lipschitz and exact; the dropout scale is one more rounding, the c 2^-24 |ref| term."""
    return 1.01 * (split_error(3) + (3 * K + 1) * U23)


def gamma_dx(N: int) -> float:
    """dX through k_linear_tc: the reduction runs over the N output features of the layer (3 N additions), and the
    weight arrives as float32(W * s), one more 2^-24 relative per term (s = 1 without dropout: exact)"""
    return 1.01 * (split_error(3) + 3 * N * U23 + U24)


def dw_launch_bounds(M: int, sms: int) -> Tuple[int, int]:
    """(largest rows_per_cta, largest CTA count) launch_linear_dw_tc can choose for M rows on ``sms`` SMs: it runs
    ctas = min(sms * per_sm, ceil(M / 64)) CTAs with 1 <= per_sm <= 4, each over ceil(slabs / ctas) 64-row slabs"""
    slabs = -(-M // 64)
    ctas_min, ctas_max = min(sms, slabs), min(4 * sms, slabs)
    return -(-slabs // ctas_min) * 64, ctas_max


def gamma_dw(M: int, sms: int) -> float:
    """k_linear_dw_tc + k_linear_dw_reduce, one output: each CTA adds 4 exact products per batch row of its range into
    one accumulator (4 rows_per_cta additions, zero rows included); the reduce adds CTAs l, l+8, ... in each of 8 lanes
    (ceil(ctas / 8) additions) and the lanes in a 3-level shuffle tree (3 additions).  A term passes through at most
    4 rows_per_cta + ceil(ctas / 8) + 3 additions, each within 2^-23 of a running sum <= S: gamma = 3 * 2^-22 +
    (4 rows_per_cta + ceil(ctas / 8) + 3) 2^-23, rows_per_cta and ctas at their largest (``dw_launch_bounds``).  The
    dropout scale is one rounding after the sum (the c 2^-24 |ref| term).  dbias is the same sum with x = 1."""
    rows, ctas = dw_launch_bounds(M, sms)
    return 1.01 * (split_error(4) + (4 * rows + -(-ctas // 8) + 3) * U23)


def gamma_sum(n: int) -> float:
    """any fp32 sum of n exact-or-rounded products in any order (the CUDA-core SGEMM routes): one rounding per product
    and n additions, 2^-23 each"""
    return 1.01 * (n + 1) * U23


def bound_violation(got, ref, S, gamma: float, c: float = 2.0) -> Optional[str]:
    """None when |got - ref| <= gamma S + c 2^-24 |ref| everywhere (NaN fails), else a description of the worst element"""
    err = (got.to(ref.device, torch.float64) - ref).abs()
    bnd = gamma * S + c * U24 * ref.abs()
    bad = ~(err <= bnd)
    if not bool(bad.any()):
        return None
    i = int(torch.argmax(torch.where(bad, err - bnd, torch.zeros_like(err)).reshape(-1).nan_to_num(math.inf)))
    return (f"{int(bad.sum())} element(s) out of bound, worst flat index {i}: |err| {float(err.reshape(-1)[i]):.3e} > "
            f"{float(bnd.reshape(-1)[i]):.3e} (ref {float(ref.reshape(-1)[i]):.6e}, S {float(S.reshape(-1)[i]):.3e})")


def ratio(got, ref, S) -> float:
    """Tier C: max |got - ref| / S over the elements with S > 0 (S = 0 elements are held to equality by Tier B)"""
    err = (got.to(ref.device, torch.float64) - ref).abs()
    pos = S > 0
    if not bool(pos.any()):
        return 0.0
    r = err[pos] / S[pos]
    return math.inf if bool(torch.isnan(r).any()) else float(r.max())


# ------------------------------------------------------------------------------------------------------------------
# Tier A: exact operands
# ------------------------------------------------------------------------------------------------------------------

def with_lo(shape, gen: torch.Generator, zero_frac: float = 0.125) -> torch.Tensor:
    """a (1 + l 2^-13), a in {-1, 1} (0 with probability zero_frac), l in {0, 1, 2, 3}: hi = a (the remainder is below
    half a TF32 ulp of 1) and lo = a l 2^-13, both TF32-exact and nonzero for l > 0"""
    a = torch.randint(0, 2, shape, generator=gen).float() * 2 - 1
    a = a * (torch.rand(shape, generator=gen) >= zero_frac).float()
    l = torch.randint(0, 4, shape, generator=gen).float()
    return a * (1 + l * LO_STEP)


def small_ints(shape, gen: torch.Generator, r: int = 2) -> torch.Tensor:
    """integers in [-r, r]: TF32-exact, lo = 0"""
    return torch.randint(-r, r + 1, shape, generator=gen).float()


def _low_bit(v: np.ndarray) -> int:
    """the exponent of the lowest set bit over the nonzero float64 values v (v all multiples of 2^that)"""
    v = v[v != 0]
    if v.size == 0:
        return 0
    m, e = np.frexp(v)
    mant = np.abs(m * 2.0 ** 53).astype(np.int64)
    low = mant & -mant
    return int((e - 53 + np.round(np.log2(low)).astype(np.int64)).min())


def exact_ok(A: torch.Tensor, B: torch.Tensor, bias: Optional[torch.Tensor] = None, margin_bits: int = 2) -> Optional[str]:
    """The Tier A property of C = A B^T (+ bias), A [M, R], B [N, R] float32, reduction over R: every element splits
    exactly (x == hi + lo, hi and lo TF32-exact, so every product the 3- or 4-product kernel forms is the exact product of
    halves); all products and the bias are multiples of one quantum q; and every output's sum of |terms| stays below
    2^(24 - margin_bits) q, so every partial sum, in any order, is an fp32 number.  None when it holds, else why not."""
    halves = []
    for name, t in (("A", A), ("B", B)):
        x = t.detach().cpu().numpy().astype(np.float32)
        hi, lo = split(x)
        if not np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), x.astype(np.float64)):
            return f"{name} does not split exactly into TF32 hi + lo"
        halves.append((hi.astype(np.float64), lo.astype(np.float64)))
    (ah, al), (bh, bl) = halves
    qa = min(_low_bit(ah), _low_bit(al) if al.any() else 1 << 30)
    qb = min(_low_bit(bh), _low_bit(bl) if bl.any() else 1 << 30)
    q = qa + qb
    if bias is not None:
        b = bias.detach().cpu().double().numpy()
        if _low_bit(b) < q:
            return "bias is not a multiple of the products' quantum"
    S = torch.from_numpy(np.abs(ah) + np.abs(al)) @ torch.from_numpy(np.abs(bh) + np.abs(bl)).t()
    if bias is not None:
        S = S + torch.from_numpy(np.abs(b))
    smax = float(S.max()) if S.numel() else 0.0
    if smax >= 2.0 ** (24 - margin_bits + q):
        return f"sum of |terms| {smax} reaches 2^{24 - margin_bits} quanta (q = 2^{q})"
    return None


@dataclass(frozen=True)
class FwdCase:
    M: int
    K: int
    N: int
    relu: bool
    bias: bool
    p: Optional[float]          # dropout after the ReLU, None: none


@dataclass(frozen=True)
class DxCase:
    M: int
    N: int                      # the layer's output features: dX reduces over them
    K: int
    relu: bool
    p: Optional[float]


@dataclass(frozen=True)
class DwCase:
    M: int
    N: int
    K: int
    relu: bool
    bias: bool
    p: Optional[float]


# the kernels' edges: M exactly at a 64-row tile boundary, one row past one, one row short of one, fewer tiles than CTAs
# (C ABI only: ops takes the SGEMM below 4096 rows), and a SASRec step's B*L
_FWD_M = [4096, 4097, 8191, 200, 4160]
_FWD_P = [None, None, 0.3, 0.5, 1.0]


def fwd_grid() -> List[FwdCase]:
    """K in {32, 64, 96, 128} x N in {16, 32, 48, 64, 80, 128} (48 and 80 padded to the wgmma width) plus N in {144, 256}
    for K <= 64 (the only K with room for the 256-wide W tiles), M, ReLU, bias and dropout rotating; and 204,800 rows at
    three shapes"""
    out, i = [], 0
    for K in (32, 64, 96, 128):
        for N in (16, 32, 48, 64, 80, 128, 144, 256):
            if N > 128 and K > 64:
                continue
            p = _FWD_P[i % len(_FWD_P)]
            out.append(FwdCase(_FWD_M[i % len(_FWD_M)], K, N, relu=p is not None or i % 2 == 0, bias=i % 3 != 1, p=p))
            i += 1
    out += [FwdCase(204800, 64, 64, True, True, None), FwdCase(204800, 32, 48, False, True, None),
            FwdCase(204800, 128, 80, True, False, None)]
    return out


def dx_grid() -> List[DxCase]:
    """every (N, K) ops.linear_bwd sends to k_linear_tc for dX (N in {32, 64, 96, 128}, K % 16 == 0 up to 256 for
    N <= 64, up to 128 otherwise), M, ReLU mask and the dropout scale (none, 2, float(1 / 0.7)) rotating"""
    ms, ps = [4096, 4097, 4159, 4160, 5000], [None, 0.5, 0.3]
    out, i = [], 0
    for N in (32, 64, 96, 128):
        for K in range(16, 257, 16):
            if K > 128 and N > 64:
                continue
            p = ps[i % 3]
            out.append(DxCase(ms[i % len(ms)], N, K, relu=p is not None or i % 2 == 1, p=p))
            i += 1
    return out


def dw_grid() -> List[DwCase]:
    """N in {4, 8, 60, 64, 68, 124, 128} (68 .. 128: a partly filled second warpgroup) x K in {16, 32, 48, 64, 80, 240}
    (wgmma widths NB = 48, 80, 256 for the K features plus the ones row); M = 64 s + 1 so the last CTA's range ends in
    a one-row slab, 204,801 rows for the smaller shapes"""
    ms, ps = [4097, 20481, 12289], [None, 0.5, 0.3]
    out, i = [], 0
    for N in (4, 8, 60, 64, 68, 124, 128):
        for K in (16, 32, 48, 64, 80, 240):
            p = ps[i % 3]
            M = 204801 if (N, K) in ((64, 64), (8, 48), (68, 16)) else ms[i % len(ms)]
            out.append(DwCase(M, N, K, relu=p is not None or i % 2 == 0, bias=i % 4 != 3, p=p))
            i += 1
    return out


def fwd_operands(M: int, K: int, N: int, lo_in: str, bias: bool, seed: int = 0):
    """Tier A operands of Y = X W^T + b: lo bits only in X (lo_in = "x") or only in W ("w"), the other operand small
    integers, so the kernel's hi*lo or lo*hi product carries them and dropping either shows.  Rows 1 and M - 1 of X are
    zero and every third bias entry is 0, so some pre-activations are exactly 0."""
    g = torch.Generator().manual_seed(seed * 1000003 + M * 7919 + K * 131 + N * 17 + (1 if lo_in == "x" else 2))
    if lo_in == "x":
        x, W = with_lo((M, K), g), small_ints((N, K), g)
    else:
        x, W = small_ints((M, K), g, r=1), with_lo((N, K), g)
    x[1 % M] = 0
    x[M - 1] = 0
    b = None
    if bias:
        b = small_ints((N,), g, r=3)
        b[::3] = 0
    return x, W, b


def dw_dense_operands(M: int, N: int, K: int, seed: int = 0):
    """Tier A operands for a long dW: dY, X, the saved output in {-1, 0, 1} (no lo bits; every partial sum an integer
    below M <= 2^18)"""
    g = torch.Generator().manual_seed(seed * 1000003 + M * 7919 + K * 131 + N * 17)
    return small_ints((M, N), g, 1), small_ints((M, K), g, 1), small_ints((M, N), g, 1)


def dw_boundary_rows(M: int, sms: int) -> List[int]:
    """batch rows at the edges the kernel partitions M along: the first and last rows, the 32-row slab and 64-row step
    edges of the first steps, and the first / last row of every CTA range any per_sm in 1..4 can give -- at most ~200"""
    rows = {0, 1, 31, 32, 33, 63, 64, 65, 127, 128, M - 2, M - 1}
    slabs = -(-M // 64)
    for per_sm in (1, 2, 3, 4):
        ctas = min(sms * per_sm, slabs)
        rpc = -(-slabs // ctas) * 64
        for c in (1, 2, ctas // 2, ctas - 1):
            for r in (c * rpc - 1, c * rpc):
                rows.add(r)
    return sorted(r for r in rows if 0 <= r < M)


def dw_sparse_operands(M: int, N: int, K: int, lo_in: str, sms: int, seed: int = 0):
    """Tier A operands for a long dW whose lo path matters: only the ``dw_boundary_rows`` are nonzero; lo bits only in
    dY (lo_in = "dy") or only in X ("x"), the other small integers; the saved output in {-1, 0, 1} on those rows"""
    g = torch.Generator().manual_seed(seed * 1000003 + M * 7919 + K * 131 + N * 17 + (1 if lo_in == "dy" else 2))
    rows = torch.tensor(dw_boundary_rows(M, sms))
    dy, x, y = torch.zeros(M, N), torch.zeros(M, K), torch.zeros(M, N)
    n = rows.numel()
    if lo_in == "dy":
        dy[rows], x[rows] = with_lo((n, N), g, zero_frac=0.0), small_ints((n, K), g, 1)
    else:
        dy[rows], x[rows] = small_ints((n, N), g, 1), with_lo((n, K), g, zero_frac=0.0)
    y[rows] = small_ints((n, N), g, 1)
    return dy, x, y


# ------------------------------------------------------------------------------------------------------------------
# fp32 emulations of the kernels' arithmetic (CPU tests of the criteria themselves)
# ------------------------------------------------------------------------------------------------------------------

def add_rz(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """fp32 a + b rounded toward zero (the worst rounding mode the error model allows)"""
    s = a.astype(np.float64) + b.astype(np.float64)
    f = s.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(s)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def add_rn(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """fp32 a + b rounded to nearest"""
    return (a + b).astype(np.float32)


def emulate_fwd(x, W, bias=None, relu=False, products=("hh", "hl", "lh"), rz=True) -> torch.Tensor:
    """k_linear_tc's arithmetic in fp32: the chosen products of TF32 halves added one term at a time into one
    accumulator (product, then k: the longest chain of roundings any order has), each addition rounded toward zero (rz)
    or to nearest; then + bias (round to nearest) and ReLU"""
    add = add_rz if rz else add_rn
    xh, xl = split(x.numpy())
    wh, wl = split(W.numpy())
    ops_ = {"hh": (xh, wh), "hl": (xh, wl), "lh": (xl, wh), "ll": (xl, wl)}
    acc = np.zeros((x.shape[0], W.shape[0]), dtype=np.float32)
    for p in products:
        a, b = ops_[p]
        for k in range(x.shape[1]):
            acc = add(acc, (a[:, k:k + 1] * b[:, k][None, :]).astype(np.float32))
    if bias is not None:
        acc = (acc + bias.numpy()[None, :]).astype(np.float32)
    if relu:
        acc = np.maximum(acc, np.float32(0))
    return torch.from_numpy(acc)


def emulate_dw(dy, x, rows_per_cta: int, products=("hh", "hl", "lh", "ll"), rz=True) -> Tuple[torch.Tensor, torch.Tensor]:
    """k_linear_dw_tc + k_linear_dw_reduce in fp32: per CTA range the chosen products of TF32 halves of dY^T and
    [X | 1], one batch row at a time, each addition rounded toward zero (rz) or to nearest; then 8 lanes over CTAs
    l, l+8, ... and a 3-level tree"""
    add = add_rz if rz else add_rn
    gh, gl = split(dy.numpy())
    xa = np.concatenate([x.numpy(), np.ones((x.shape[0], 1), dtype=np.float32)], axis=1)
    xh, xl = split(xa)
    ops_ = {"hh": (gh, xh), "hl": (gh, xl), "lh": (gl, xh), "ll": (gl, xl)}
    M, N, K1 = dy.shape[0], dy.shape[1], xa.shape[1]
    parts = []
    for m0 in range(0, M, rows_per_cta):
        acc = np.zeros((N, K1), dtype=np.float32)
        for m in range(m0, min(M, m0 + rows_per_cta)):
            for p in products:
                a, b = ops_[p]
                acc = add(acc, (a[m][:, None] * b[m][None, :]).astype(np.float32))
        parts.append(acc)
    lanes = []
    for l in range(8):
        a = np.zeros((N, K1), dtype=np.float32)
        for c in range(l, len(parts), 8):
            a = add(a, parts[c])
        lanes.append(a)
    for step in (1, 2, 4):
        lanes = [add(lanes[l], lanes[l ^ step]) for l in range(8)]
    out = torch.from_numpy(lanes[0])
    return out[:, :-1].contiguous(), out[:, -1].contiguous()


# ------------------------------------------------------------------------------------------------------------------
# the Tier A operands of each grid case (shared by the GPU tests and the CPU check of their representability)
# ------------------------------------------------------------------------------------------------------------------

def fwd_case_operands(case: FwdCase, lo_in: str):
    """(x, W, bias) of a forward case, lo bits in "x" or "w"; exact_ok(x, W, bias) holds"""
    return fwd_operands(case.M, case.K, case.N, lo_in, case.bias)


def dx_case_operands(case: DxCase, lo_in: str):
    """(dy, W, y_relu) of a dX case, lo bits in "dy" or "w": the kernel computes (dy o [y > 0]) (W^T)^T, so the forward's
    operands with X = dy and the forward weight = W^T; the saved output in {0, 1} (None without ReLU)"""
    dy, Wt, _ = fwd_operands(case.M, case.N, case.K, "x" if lo_in == "dy" else "w", False, seed=1)
    g = torch.Generator().manual_seed(case.M * 31 + case.N * 7 + case.K)
    y = small_ints((case.M, case.N), g, 1).clamp_min(0) if case.relu else None
    return dy, Wt.t().contiguous(), y


def dw_small_operands(M: int, N: int, K: int, lo_in: str):
    """(dy, x, y_relu) for the C ABI at M <= 255: every row dense, lo bits only in dY ("dy") or only in X ("x")"""
    g = torch.Generator().manual_seed(M * 7919 + K * 131 + N * 17 + (1 if lo_in == "dy" else 2))
    if lo_in == "dy":
        dy, x = with_lo((M, N), g), small_ints((M, K), g, 1)
    else:
        dy, x = small_ints((M, N), g, 1), with_lo((M, K), g)
    return dy, x, small_ints((M, N), g, 1)


def dw_exact_terms(dy, x, y_relu):
    """the A [N, M] and B [K + 1, M] of the dW kernel's contraction: (dy o [y > 0])^T and [x | 1]^T"""
    g = dy if y_relu is None else dy * (y_relu > 0).float()
    return g.t().contiguous(), torch.cat([x, torch.ones(x.shape[0], 1)], dim=1).t().contiguous()
