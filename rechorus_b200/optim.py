"""Optimizer for the ``model.optimizer`` seam of the reference's runner (helpers/BaseRunner.py:176-177,193,206).

``BaseRunner.fit`` only builds ``torch.optim.<name>`` when ``model.optimizer is None``; an object with
``zero_grad()`` / ``step()`` placed there beforehand is used as-is.  ``RowSparseOptimizer`` is that object:

* embedding tables in 'fused' mode (rechorus_b200.ops.set_table_mode): the contribution streams parked by the
  backward pass are reduced per unique row and the SGD/Adam/Adagrad update is applied in the same kernel
  (b2r_segment_apply mode 2).  The update is *row-sparse / lazy*: rows the batch did not touch do not move.
  This is NOT what the reference's dense ``torch.optim.Adam`` does (there the moments keep moving untouched
  rows and L2 decays them every step); it is the semantics of ``torch.optim.SparseAdam`` and of production
  recommender training.  Keep tables in 'dense' mode to reproduce the reference exactly, or pass ``exact_dense=True``
  for the reference's dense Adam results at row-sparse cost.
* every other parameter (and tables left in 'dense' mode) gets the exact dense torch.optim formula
  (b2r_dense_optim), with the reference's two parameter groups: names containing 'bias' have weight_decay 0
  (models/BaseModel.py:64-73).
"""
from __future__ import annotations

from typing import Dict, List

import torch

from . import lib as _lib
from . import ops

_KIND = {"SGD": _lib.OPT_SGD, "Adam": _lib.OPT_ADAM, "Adagrad": _lib.OPT_ADAGRAD}
_DEFAULT_EPS = {"SGD": 0.0, "Adam": 1e-8, "Adagrad": 1e-10}


class RowSparseOptimizer:
    def __init__(self, model: torch.nn.Module, name: str = "Adam", lr: float = 1e-3, l2: float = 0.0,
                 betas=(0.9, 0.999), eps: float | None = None, exact_dense: bool = False, device_clock: bool = False):
        """exact_dense (Adam only): keep the row-sparse cost but reproduce the reference's dense torch.optim.Adam --
        every fused table gets a per-row "up to date as of step" stamp, the rows a forward reads are advanced through
        the steps they skipped before it reads them (``before_forward``, called by every kernel-backed model's
        forward and by the single-call BPRMF step), the rows an update writes are stamped with its step, and
        ``flush()`` brings the whole table up to date (oracle.LazyExactAdam).  The catch-up deduplicates the raw ids
        on the device (b2r_adam_exact_catch_up), so the mode adds no host synchronisation to a training step.
        Fused tables must be 32, 64 or 128 wide, the widths of the catch-up and apply kernels."""
        if name not in _KIND:
            raise ValueError(f"optimizer {name!r} not supported by the fused path (have {sorted(_KIND)})")
        if exact_dense and name != "Adam":
            raise ValueError("exact_dense applies to Adam only (row-sparse SGD without weight decay already is exact)")
        self.exact_dense = bool(exact_dense)
        if exact_dense and device_clock:
            raise ValueError("exact_dense keeps its bookkeeping on the host: not available with device_clock")
        # device_clock: the step count and Adam's bias corrections live in a 4-float device array advanced by a one-thread
        # kernel inside step() (b2r_optim_tick); the update kernels read them from there, so a step enqueued once -- or
        # captured in a CUDA graph (rechorus_b200.graph.GraphedStep) -- stays correct when replayed
        self.clock = None
        self._want_clock = bool(device_clock)
        self.name, self.kind = name, _KIND[name]
        self.lr, self.l2, self.betas = float(lr), float(l2), (float(betas[0]), float(betas[1]))
        self.eps = _DEFAULT_EPS[name] if eps is None else float(eps)
        self.t = 0
        self._flushed_at = 0                  # exact_dense: the step every row was last brought up to by flush()
        self.model = model
        self._entries: List[dict] = []
        for pname, p in model.named_parameters():
            if not p.requires_grad:
                continue
            wd = 0.0 if "bias" in pname else self.l2
            e = {"name": pname, "p": p, "wd": wd, "m": None, "v": None, "state_ld": 0}
            if self.kind == _lib.OPT_ADAM and ops.table_mode(p) == "fused" and p.dim() == 2:
                # row-sparse Adam touches m[row] and v[row] together: keep them interleaved per row
                # ([n_rows][2][d]) so each row's state is one contiguous 2*4d-byte burst in HBM
                mv = torch.zeros((p.shape[0], 2, p.shape[1]), dtype=p.dtype, device=p.device)
                e["mv"], e["m"], e["v"], e["state_ld"] = mv, mv[:, 0, :], mv[:, 1, :], 2 * p.shape[1]
                if self.exact_dense:
                    if p.shape[1] not in (32, 64, 128):
                        raise ValueError(f"exact_dense: table {pname} is {p.shape[1]} wide; the exact dense-Adam "
                                         "catch-up runs on tables 32, 64 or 128 wide")
                    e["last"] = torch.zeros(p.shape[0], dtype=torch.int32, device=p.device)
            else:
                if self.kind == _lib.OPT_ADAM:
                    e["m"] = torch.zeros_like(p.data)
                if self.kind != _lib.OPT_SGD:
                    e["v"] = torch.zeros_like(p.data)
            self._entries.append(e)

    # -- exact dense-Adam bookkeeping (exact_dense=True) ----------------------------------------------------
    def _cfg(self, e: dict):
        import types
        return types.SimpleNamespace(lr=self.lr, betas=self.betas, eps=self.eps, weight_decay=e["wd"])

    def before_forward(self, param: torch.Tensor, ids: torch.Tensor, ignore_id: int = -1) -> None:
        """bring the rows a forward pass is about to read (``ids``, any shape, repeats allowed; ``ignore_id`` e.g. the
        padding id of histories is skipped) up to the current step (no-op unless exact_dense)"""
        if not self.exact_dense:
            return
        e = self.entry(param)
        if "last" in e and self.t > 0:
            ops.adam_exact_catch_up(e["p"].data, e["m"], e["v"], e["last"], ids, self.t, self._cfg(e),
                                    ignore_id=ignore_id, ignore_n=ids.numel() if ignore_id >= 0 else 0,
                                    state_ld=e["state_ld"])

    def flush(self) -> None:
        """bring every row of every exact table up to the current step (before evaluation, saving, reading weights);
        a no-op when no step was taken since the last flush"""
        if not self.exact_dense or self._flushed_at == self.t:
            return
        for e in self._entries:
            if "last" in e:
                ops.adam_exact_advance(e["p"].data, e["m"], e["v"], e["last"], self.t, self._cfg(e),
                                       state_ld=e["state_ld"])
        self._flushed_at = self.t

    # -- torch.optim-like surface used by BaseRunner.fit ------------------------------------------------
    def zero_grad(self, set_to_none: bool = True) -> None:
        for e in self._entries:
            p = e["p"]
            p.grad = None
            pend = getattr(p, "_b2r_pending", None)
            if pend:
                pend.clear()

    def _opt(self, wd: float, state_ld: int = 0) -> _lib.Optim:
        b1, b2 = self.betas
        t = max(self.t, 1)
        clock = self.clock.data_ptr() if self.clock is not None else None
        return _lib.Optim(self.kind, self.lr, b1, b2, self.eps, wd, 1.0 - b1 ** t, 1.0 - b2 ** t, state_ld, clock)

    def _tick(self) -> None:
        """one optimizer step begins: host counter, and the device clock when there is one"""
        self.t += 1
        if self._want_clock:
            if self.clock is None:
                dev = next(e["p"].device for e in self._entries)
                self.clock = torch.zeros(4, dtype=torch.float32, device=dev)
                if self.t > 1:                                   # resume from a host-counted history
                    self.clock[0] = float(self.t - 1)
            from . import lib as L_
            L_.check(L_.load().b2r_optim_tick(self.clock.data_ptr(), self.lr, self.betas[0], self.betas[1],
                                              torch.cuda.current_stream().cuda_stream), "b2r_optim_tick")

    def sync_clock(self) -> int:
        """after graph replays the host counter is stale: read the step count back from the device clock"""
        if self.clock is not None:
            self.t = int(round(float(self.clock[0].item())))
        return self.t

    @torch.no_grad()
    def step(self) -> None:
        self._tick()
        for e in self._entries:
            p = e["p"]
            pend = getattr(p, "_b2r_pending", None)
            if ops.table_mode(p) == "fused" and pend is not None:
                if not pend:
                    continue
                if len(pend) > 2:
                    raise _lib.B200RecError(f"{e['name']}: more than two gradient streams into one table")
                # a stream with an ignore id (padding) must come first: the plan drops ignore_id only in a prefix
                pend.sort(key=lambda x: 0 if x[2] >= 0 else 1)
                if len(pend) == 2 and pend[1][2] >= 0:
                    raise _lib.B200RecError(f"{e['name']}: two padded gradient streams into one table")
                ids = pend[0][0] if len(pend) == 1 else torch.cat([pend[0][0], pend[1][0]])
                ign = pend[0][2]
                if "last" in e:
                    # exact dense-Adam mode: the rows about to be updated must stand at step t-1 (they do already:
                    # the forward that parked these streams caught them up) and are stamped t, the step the update
                    # below applies; the plan's padding rule (ignore id in the first stream only) is the catch-up's
                    ops.adam_exact_catch_up(p.data, e["m"], e["v"], e["last"], ids, self.t - 1, self._cfg(e),
                                            stamp=self.t, ignore_id=ign, ignore_n=pend[0][0].numel() if ign >= 0 else 0,
                                            state_ld=e["state_ld"])
                plan = ops.make_plan(ids, p.shape[0], p.shape[1], ign, pend[0][0].numel() if ign >= 0 else 0)
                plan.apply_optimizer(p.data, e["m"], e["v"], self._opt(e["wd"], e["state_ld"]), [x[1] for x in pend])
                pend.clear()
            elif p.grad is not None:
                if p.grad.is_sparse:
                    raise _lib.B200RecError(f"{e['name']}: sparse .grad -- use table mode 'fused' or 'dense' "
                                            "with RowSparseOptimizer, or torch.optim.SparseAdam")
                g = p.grad if p.grad.is_contiguous() else p.grad.contiguous()
                if e["state_ld"]:
                    raise _lib.B200RecError(f"{e['name']}: table left 'fused' mode after the optimizer was built")
                ops.dense_optim(p.data, g, e["m"], e["v"], self._opt(e["wd"]))

    def entry(self, param: torch.Tensor) -> dict:
        """state record (m, v, weight decay) of one parameter -- used by the models' C-side fused step"""
        for e in self._entries:
            if e["p"] is param:
                return e
        raise KeyError("parameter is not managed by this optimizer")

    def advance(self) -> int:
        """count one optimizer step taken outside ``step()`` (the C-side whole-step entry points)"""
        self._tick()
        return self.t

    # -- checkpointing (the reference saves no optimizer state; kept for completeness) -------------------
    def state_dict(self) -> Dict:
        return {"t": self.t, "name": self.name,
                "state": {e["name"]: {"m": e["m"], "v": e["v"]} for e in self._entries}}

    def load_state_dict(self, sd: Dict) -> None:
        self.t = int(sd["t"])
        self._flushed_at = -1
        for e in self._entries:
            st = sd["state"].get(e["name"])
            if st is None:
                continue
            for k in ("m", "v"):
                if e[k] is not None and st[k] is not None:
                    e[k].copy_(st[k])
