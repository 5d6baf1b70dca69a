"""Float64 restatement of the row-sparse table-gradient contract (b2r_grad_source in include/b200rec.h) and of the
lazy SGD / Adam / Adagrad row update, for tests only.

Position p of a plan adds coef[p] * src[row(p)] to table row id[p], where row(p) = src_id[p // div] when src_id is
given and p // div otherwise, and src row r starts at float offset + r * ld.  A plan may take two sources: positions
[0, n0) are the first one's, [n0, n0 + n1) the second one's.  Positions in [0, ignore_n) holding ignore_id contribute
nothing; an id outside [0, n_rows) is clamped to row 0 and counted, as the kernels do.  A row is touched when a
position that is not dropped names it, whatever its coefficient.

The optimizer constants are the float32 values the kernels use (make_optk in csrc/common.cuh), promoted to float64, so
a comparison measures the kernels' arithmetic and not how the constants were rounded.  Works on CPU or CUDA tensors.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np
import torch

U = 2.0 ** -24          # unit roundoff of float32
U64 = 2.0 ** -53


def gamma(k, u: float = U):
    """gamma(k) = k u / (1 - k u): the classic bound on the relative error of k chained float operations"""
    k = k.to(torch.float64) if isinstance(k, torch.Tensor) else float(k)
    return k * u / (1.0 - k * u)


@dataclass
class Stream:
    """One contribution source.  ``src`` is any float32 tensor; its storage is addressed as the kernels address the
    pointer they are given: row r of the source is storage[offset + r * ld : offset + r * ld + d]."""
    src: torch.Tensor
    n: int
    ld: int
    offset: int = 0
    coef: Optional[torch.Tensor] = None
    src_id: Optional[torch.Tensor] = None
    div: int = 1

    def contributions(self, d: int) -> torch.Tensor:
        """[n, d] float64: coef[p] * src[row(p)] for every position of this stream (exact: a float32 product)"""
        dev = self.src.device
        p = torch.arange(self.n, device=dev, dtype=torch.int64)
        r = p // max(1, int(self.div))
        if self.src_id is not None:
            r = self.src_id.to(dev)[r]
        n_src = int(r.max()) + 1 if self.n else 0
        rows = torch.as_strided(self.src, (n_src, d), (self.ld, 1), self.offset)
        out = rows.to(torch.float64)[r]
        if self.coef is not None:
            out *= self.coef.to(dev, torch.float64)[:self.n].unsqueeze(1)
        return out


@dataclass
class TableGrad:
    rows: torch.Tensor       # [nu] int64, ascending: the touched rows
    grad: torch.Tensor       # [nu, d] float64 gradient of each touched row
    absum: torch.Tensor      # [nu, d] float64 sum over the row's contributions of |coef * src|
    count: torch.Tensor      # [nu] int64 contributions of each touched row
    n_bad: int               # out-of-range ids (clamped to row 0)

    def bound(self, dense0: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[nu, d] float64: the largest |out - (dense0 + grad)| any summation order of the row's contributions in float32
        (fused multiply-adds, partial sums combined in any order) followed by the add into dense0 can give:
        gamma(k + 1) (A + |dense0|), plus the float64 reference's own rounding"""
        a = self.absum if dense0 is None else self.absum + dense0.to(torch.float64).abs()
        k = (self.count + 1).unsqueeze(1)
        return (gamma(k) + gamma(k, U64)) * a


def table_grad(ids: torch.Tensor, n_rows: int, d: int, streams: Sequence[Stream], ignore_id: int = -1,
               ignore_n: int = 0) -> TableGrad:
    ids = ids.reshape(-1).to(torch.int64)
    n = ids.numel()
    if sum(s.n for s in streams) != n:
        raise ValueError("streams do not cover the ids")
    p = torch.arange(n, device=ids.device)
    drop = (p < ignore_n) & (ids == ignore_id)
    bad = ~drop & ((ids < 0) | (ids >= n_rows))
    key = torch.where(bad, torch.zeros_like(ids), ids)[~drop]
    contrib = torch.cat([s.contributions(d).to(ids.device) for s in streams])[~drop]
    rows, inv, count = torch.unique(key, sorted=True, return_inverse=True, return_counts=True)
    grad = torch.zeros((rows.numel(), d), dtype=torch.float64, device=ids.device)
    absum = torch.zeros_like(grad)
    grad.index_add_(0, inv, contrib)
    absum.index_add_(0, inv, contrib.abs())
    return TableGrad(rows, grad, absum, count, int(bad.sum()))


# ---- lazy optimizer update, float64 on the kernels' float32 constants -------------------------------------------------

def f32(x: float) -> float:
    return float(np.float32(x))


@dataclass
class OptConsts:
    """make_optk (csrc/common.cuh) from the fields of b2r_optim: beta, 1 - beta (rounded from the float32 beta), the
    step size float32(lr / bc1) and float32(1 / sqrt(bc2))"""
    kind: int               # 0 SGD, 1 Adam, 2 Adagrad
    lr: float
    beta1: float
    beta2: float
    eps: float
    wd: float
    omb1: float
    omb2: float
    step: float
    isb2: float

    @classmethod
    def of(cls, kind, lr, beta1, beta2, eps, wd, bc1=1.0, bc2=1.0) -> "OptConsts":
        lr, beta1, beta2, eps, wd, bc1, bc2 = (f32(x) for x in (lr, beta1, beta2, eps, wd, bc1, bc2))
        step = f32(lr / bc1) if kind == 1 and bc1 != 0.0 else lr
        isb2 = f32(1.0 / math.sqrt(bc2)) if kind == 1 and bc2 > 0.0 else 1.0
        return cls(kind, lr, beta1, beta2, eps, wd, f32(1.0 - beta1), f32(1.0 - beta2), step, isb2)


def grad_with_decay(K: OptConsts, G: torch.Tensor, W0: torch.Tensor) -> torch.Tensor:
    """g = G + wd * W0 (coupled L2, as torch.optim), float64"""
    return G.to(torch.float64) + K.wd * W0.to(torch.float64)


def adam_moments(K: OptConsts, m0, v0, g):
    m0, v0 = m0.to(torch.float64), v0.to(torch.float64)
    return K.beta1 * m0 + K.omb1 * g, K.beta2 * v0 + K.omb2 * g * g


def adam_weight(K: OptConsts, W0, m, v):
    """W0 - step * m / (sqrt(v) * isb2 + eps) from given moments (the kernel's own, so W is checked apart from them)"""
    m, v = m.to(torch.float64), v.to(torch.float64)
    return W0.to(torch.float64) - K.step * m / (v.sqrt() * K.isb2 + K.eps)


def adagrad_state(K: OptConsts, v0, g):
    return v0.to(torch.float64) + g * g


def adagrad_weight(K: OptConsts, W0, v, g):
    return W0.to(torch.float64) - K.lr * g / (v.to(torch.float64).sqrt() + K.eps)


def sgd_weight(K: OptConsts, W0, g):
    return W0.to(torch.float64) - K.lr * g
