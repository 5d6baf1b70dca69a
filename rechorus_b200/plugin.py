"""The reference's model plugin contract, re-hosted on the sm_90a kernels.

ReChorus discovers a model class by name and drives it through a fixed surface (SURVEY.md section 8b1):
``parse_model_args`` / ``__init__(args, corpus)`` / ``forward(feed_dict) -> {'prediction': [B, C]}`` /
``loss(out_dict)`` / ``customize_parameters`` / ``save_model`` / ``load_model`` / inner ``Dataset``.
This module provides that surface twice:

* stand-alone classes (``BPRMF``, ``NeuMF``, ``SASRec``) usable without the reference checkout -- this is what
  the tests, ``bench.py`` and ``rechorus_b200.runner.BaseRunner`` use (they must not need the reference tree);
* kernel *mixins* (``BPRMFKernels`` ...) that ``rechorus_b200.overlay`` grafts onto the reference's own
  ``GeneralModel`` / ``SequentialModel`` so the reference's unchanged ``src/main.py`` runs them.

State-dict keys and shapes equal the reference's (SURVEY.md A.5) so ``.pt`` checkpoints interchange.
There is no CPU path: calling ``forward`` with CPU tensors raises.
"""
from __future__ import annotations

import logging
import os
from typing import Dict, List

import numpy as np
import torch
import torch.nn as nn
from torch.nn.utils.rnn import pad_sequence
from torch.utils.data import Dataset as TorchDataset

from . import ops

# ======================================================================================================
# kernel mixins: parameters + forward/loss/inference, independent of which GeneralModel base hosts them
# ======================================================================================================


# SASRec's last block runs for the one query per sequence whose output is used (exact); tests set this False for the
# full last block, the reference they compare against.
_SASREC_LASTQ = True


class _KernelModelMixin:
    """Shared by every kernel-backed model: table registry + loss + optional inference hook."""

    def _register_tables(self, *params: nn.Parameter, mode: str = "dense") -> None:
        self.__dict__["_b2r_tables"] = list(params)
        for p in params:
            ops.set_table_mode(p, mode)

    def sparse_tables(self) -> List[nn.Parameter]:
        return list(getattr(self, "_b2r_tables", []))

    def set_table_mode(self, mode: str) -> None:
        """'dense' (exact reference semantics with stock torch.optim), 'sparse' (torch sparse grads) or
        'fused' (row-sparse fused optimizer, rechorus_b200.optim.RowSparseOptimizer)."""
        for p in self.sparse_tables():
            ops.set_table_mode(p, mode)

    # ``model.optimizer`` is the seam helpers/BaseRunner.py:176-177 checks: when the tables are in 'fused' mode
    # the (reference's or our) runner must find a RowSparseOptimizer there instead of building torch.optim,
    # which would silently skip parameters whose .grad stays None.  Built lazily, after main.py:68 moved the
    # model to the device.
    @property
    def optimizer(self):
        opt = self.__dict__.get("_b2r_optimizer")
        if opt is None and any(ops.table_mode(p) == "fused" for p in self.sparse_tables()):
            tables = self.sparse_tables()
            if tables and tables[0].is_cuda:
                from .optim import RowSparseOptimizer
                a = self.__dict__.get("_b2r_args")
                opt = RowSparseOptimizer(self, getattr(a, "optimizer", "Adam"), lr=getattr(a, "lr", 1e-3),
                                         l2=getattr(a, "l2", 0.0), exact_dense=bool(getattr(a, "exact_adam", 0)),
                                         device_clock=bool(getattr(a, "graph_step", 0)))
                self.__dict__["_b2r_optimizer"] = opt
        return opt

    @optimizer.setter
    def optimizer(self, value):
        self.__dict__["_b2r_optimizer"] = value

    # Out-of-range ids: the reference's nn.Embedding raises IndexError inside forward (BPRMF.py:39-40); the kernels
    # clamp the id and count it on the device.  Every runner (the reference's unchanged BaseRunner included) switches
    # the model between train() and eval() around each fit / predict (BaseRunner.py:179,231), so the counter is polled
    # there: one synchronising 4-byte read per phase switch, and a bad id surfaces as the same IndexError.
    def train(self, mode: bool = True):
        tables = self.sparse_tables()
        if tables and tables[0].is_cuda:
            ops.poll_ids(tables[0].device)
        return super().train(mode)

    # Dropout (NeuMF.py:70-72, layers.py:113-117) runs inside the Linear / residual-LayerNorm kernels with a counter-based
    # mask (include/b200rec.h, b2r_dropout).  Its seed is torch.initial_seed() at construction -- read, not drawn, so the
    # reference's CPU RNG streams stay in step -- and its step counter lives on the device, ticked once per training
    # forward (so a captured CUDA graph advances it on every replay).  Neither is part of the state_dict.
    def _dropout_init(self) -> None:
        self.__dict__["_b2r_drop_seed"] = torch.initial_seed()

    def _dropout_state(self, device) -> "ops.DropoutState":
        st = self.__dict__.get("_b2r_drop_state")
        if st is None:
            seed = self.__dict__.get("_b2r_drop_seed")
            st = ops.DropoutState(torch.initial_seed() if seed is None else seed, device)
            self.__dict__["_b2r_drop_state"] = st
        return st

    def _dropout_snapshot(self, device):
        """the forward's {seed, step} snapshot (one tick), or None when no dropout applies (p = 0 or eval mode)"""
        if not (self.training and self.dropout > 0):
            return None
        return self._dropout_state(device).tick()

    def dropout_rng_state(self):
        """(seed, step) of the dropout stream: the next training forward draws its masks at this step"""
        dev = next(self.parameters()).device
        return self._dropout_state(dev).get()

    def set_dropout_rng_state(self, seed: int, step: int) -> None:
        self._dropout_state(next(self.parameters()).device).set(seed, step)

    # models/BaseModel.py:175-189
    def loss(self, out_dict: dict) -> torch.Tensor:
        return ops.bpr_loss(out_dict["prediction"])

    # helpers/BaseRunner.py:237 looks for this optional hook: scoring without building an autograd graph
    def inference(self, feed_dict: dict) -> dict:
        with torch.no_grad():
            return self.forward(feed_dict)

    # Evaluation on the device (SURVEY.md §8 f2).  Models whose candidate score is a dot product with an item-table
    # row return (query rows [B, d], item table) here; others return None and are ranked from their predictions.
    def query_rows(self, feed_dict: dict):
        return None

    def eval_ranks(self, feed_dict: dict, mask_row=None, mask_item=None, clicked=None) -> torch.Tensor:
        """int64 [B] ranks of the ground-truth item (helpers/BaseRunner.py:63) for one evaluation batch, computed
        on the device.  Under the test_all protocol (candidates = [target] + arange(1, n_items),
        BaseModel.py:194-198) a dot-product model is ranked without materialising the [B, n_items] scores;
        (mask_row, mask_item) are the (batch row, item id) pairs BaseRunner.py:244-251 would set to -inf.
        ``clicked`` (ops.ClickedSets, test_all only) names those pairs instead as the clicked items of each row's user;
        a dot-product model then needs only column 0 of feed_dict["item_id"]."""
        with torch.no_grad():
            self._flush_exact()
            item_id = feed_dict["item_id"]
            test_all = bool(getattr(self, "test_all", 0))
            if clicked is not None and test_all and self.has_query_rows():
                q, table = self.query_rows(feed_dict)
                return ops.rank_all_items_clicked(q, table, item_id[:, 0], feed_dict["user_id"], clicked)
            qr = self.query_rows(feed_dict) if test_all else None
            if qr is not None and item_id.shape[1] == self.item_num:
                q, table = qr
                return ops.rank_all_items(q, table, item_id[:, 0], mask_row, mask_item)
            if clicked is not None and test_all and item_id.shape[1] != self.item_num:
                raise ValueError(f"test_all candidate lists have {self.item_num} columns, got {item_id.shape[1]}")
            pred = self.forward(feed_dict)["prediction"]
            if clicked is not None and test_all:
                pred = ops.mask_clicked(pred.contiguous(), feed_dict["user_id"], clicked)
            if mask_row is not None and mask_row.numel() > 0:
                pred = pred.clone()
                pred[mask_row, mask_item] = float("-inf")
            return ops.gt_rank(pred)

    def _flush_exact(self) -> None:
        opt = self.__dict__.get("_b2r_optimizer")
        if getattr(opt, "exact_dense", False) and not self.training:
            opt.flush()                     # exact dense-Adam mode: ranks and lists must see rows advanced through skipped steps

    def _exact_catch_up(self, *reads) -> None:
        """Exact dense-Adam mode (RowSparseOptimizer(exact_dense=True)): a training forward first advances the rows it is
        about to read -- each of ``reads`` is (table, ids) or (table, ids, ignore id) -- through the optimizer steps they
        skipped, on the device and without a host synchronisation; an eval-mode forward (the host predict route through
        ``inference``) flushes every table instead.  A no-op in the lazy mode."""
        opt = self.__dict__.get("_b2r_optimizer")
        if not getattr(opt, "exact_dense", False):
            return
        if self.training:
            for r in reads:
                opt.before_forward(*r)
        else:
            opt.flush()

    def has_query_rows(self) -> bool:
        """whether this model scores candidates as dot products with item-table rows (query_rows is overridden)"""
        return type(self).query_rows is not _KernelModelMixin.query_rows

    def recommend(self, feed_dict: dict, k: int, clicked=None):
        """The top-k' recommendation lists (k' = min(k, C)) of one evaluation batch on the device: (item ids int64 [B, k'],
        scores float32 [B, k']) in the order of main.py:117-132's stable sort of (item_id, prediction) pairs
        (include/b200rec.h).  Under test_all the candidates are [target] + arange(1, n_items) with the items of
        ``clicked`` (ops.ClickedSets) masked to -inf (BaseRunner.py:244-251); column 0 of feed_dict["item_id"] is the
        target and a dot-product model needs no other column (ops.topk_all_items scores the catalogue itself)."""
        with torch.no_grad():
            self._flush_exact()
            item_id = feed_dict["item_id"]
            test_all = bool(getattr(self, "test_all", 0))
            if test_all and clicked is None:
                raise ValueError("recommend under test_all needs the clicked sets (ops.ClickedSets) to mask")
            if test_all and self.has_query_rows():
                q, table = self.query_rows(feed_dict)
                return ops.topk_all_items(q, table, item_id[:, 0], feed_dict["user_id"], clicked, k)
            if test_all and item_id.shape[1] != self.item_num:
                raise ValueError(f"test_all candidate lists have {self.item_num} columns, got {item_id.shape[1]}")
            pred = self.forward(feed_dict)["prediction"].contiguous()
            if test_all:
                ops.mask_clicked(pred, feed_dict["user_id"], clicked)
            cols, scores = ops.topk_rows(pred, k)
            return item_id.gather(1, cols), scores


class BPRMFKernels(_KernelModelMixin):
    """models/general/BPRMF.py:18-45 (BPRMFBase) on K1/K2."""

    @staticmethod
    def parse_model_args(parser):
        parser.add_argument("--emb_size", type=int, default=64, help="Size of embedding vectors.")
        parser.add_argument("--table_mode", type=str, default="dense",
                            help="embedding gradient form: dense | sparse | fused (see rechorus_b200.ops)")
        return parser

    def _base_init(self, args, corpus):
        self.__dict__["_b2r_args"] = args
        self.emb_size = args.emb_size
        if self.emb_size % 4 != 0:
            raise ValueError("rechorus_b200 kernels need emb_size % 4 == 0")
        self._base_define_params()
        self.apply(self.init_weights)
        self._register_tables(self.u_embeddings.weight, self.i_embeddings.weight,
                              mode=getattr(args, "table_mode", "dense"))

    def _base_define_params(self):
        # same module/parameter names as BPRMF.py:31-32 -> identical state_dict keys
        self.u_embeddings = nn.Embedding(self.user_num, self.emb_size)
        self.i_embeddings = nn.Embedding(self.item_num, self.emb_size)

    def forward(self, feed_dict):
        self.check_list = []
        u_ids = feed_dict["user_id"]        # [B]
        i_ids = feed_dict["item_id"]        # [B, C]
        self._exact_catch_up((self.u_embeddings.weight, u_ids), (self.i_embeddings.weight, i_ids))
        u = ops.embedding(self.u_embeddings.weight, u_ids)            # [B, d]   (gather kernel)
        pred = ops.score(u, self.i_embeddings.weight, i_ids)          # [B, C]   (gather + dot kernel)
        out = {"prediction": pred.view(feed_dict["batch_size"], -1)}
        if getattr(self, "_b2r_vectors", False):
            # BPRMFBase.forward also returns the vectors (BPRMF.py:43-45) -- re-rankers stack them under a base ranker
            # (BaseRerankerModel.py:82-83).  The plain BPRMF drops them (:60-62), the Impression variant keeps them.
            out["u_v"] = u.unsqueeze(1).expand(-1, i_ids.shape[1], -1)
            out["i_v"] = ops.embedding(self.i_embeddings.weight, i_ids)
        return out

    def query_rows(self, feed_dict):
        with torch.no_grad():
            return ops.embedding(self.u_embeddings.weight, feed_dict["user_id"]), self.i_embeddings.weight

    def train_step(self, feed_dict, next_feed_dict=None) -> torch.Tensor:
        """One whole training step (forward, BPR loss, backward, row-sparse optimizer update) enqueued by a
        single C call (b2r_bprmf_train_step) -- the body of helpers/BaseRunner.py:193-206 for this model.
        Needs ``self.optimizer`` to be a ``RowSparseOptimizer``.  ``next_feed_dict`` (optional) is the next
        batch, already on the device: its index plan is prefetched while this step runs.  Returns the loss as a
        device scalar."""
        if (self.emb_size not in (32, 64, 128)
                or not ops.DirectPlan.available(feed_dict["item_id"].numel(), self.item_num)):
            # no plan/apply kernel for this width, or a batch too large for the step's index plans: same step through
            # the autograd nodes
            self.optimizer.zero_grad()
            loss = self.loss(self.forward(feed_dict))
            loss.backward()
            self.optimizer.step()
            return loss.detach()
        nu = ni = None
        if next_feed_dict is not None:
            nu, ni = next_feed_dict["user_id"], next_feed_dict["item_id"]
        return ops.bprmf_train_step(self.u_embeddings.weight, self.i_embeddings.weight, self.optimizer,
                                    feed_dict["user_id"], feed_dict["item_id"], nu, ni)


class NeuMFKernels(_KernelModelMixin):
    """models/general/NeuMF.py:22-76 on the library kernels: four row-sparse tables, GMF branch folded into the
    gather+dot kernel (pred_mf = <w_mf * mf_u[b], mf_i[id]>), MLP tower on the fp32 SGEMM."""

    @staticmethod
    def parse_model_args(parser):
        parser.add_argument("--emb_size", type=int, default=64, help="Size of embedding vectors.")
        parser.add_argument("--layers", type=str, default="[64]", help="Size of each layer.")
        parser.add_argument("--table_mode", type=str, default="dense",
                            help="embedding gradient form: dense | sparse | fused (see rechorus_b200.ops)")
        return parser

    def _neumf_init(self, args, corpus):
        import ast
        self.__dict__["_b2r_args"] = args
        self.emb_size = args.emb_size
        if self.emb_size % 4 != 0:
            raise ValueError("rechorus_b200 kernels need emb_size % 4 == 0")
        self.layers = list(ast.literal_eval(args.layers))      # the reference eval()s this string (NeuMF.py:38)
        self._dropout_init()
        self._define_params()
        self.apply(self.init_weights)
        self._register_tables(self.mf_u_embeddings.weight, self.mf_i_embeddings.weight,
                              self.mlp_u_embeddings.weight, self.mlp_i_embeddings.weight,
                              mode=getattr(args, "table_mode", "dense"))

    def _define_params(self):
        # same module names as NeuMF.py:42-54 -> identical state_dict keys
        d = self.emb_size
        self.mf_u_embeddings = nn.Embedding(self.user_num, d)
        self.mf_i_embeddings = nn.Embedding(self.item_num, d)
        self.mlp_u_embeddings = nn.Embedding(self.user_num, d)
        self.mlp_i_embeddings = nn.Embedding(self.item_num, d)
        self.mlp = nn.ModuleList([])
        pre = 2 * d
        for width in self.layers:
            self.mlp.append(nn.Linear(pre, width))
            pre = width
        self.dropout_layer = nn.Dropout(p=self.dropout)
        self.prediction = nn.Linear(pre + d, 1, bias=False)

    def forward(self, feed_dict):
        self.check_list = []
        u_ids = feed_dict["user_id"]        # [B]
        i_ids = feed_dict["item_id"]        # [B, C]
        B, C = i_ids.shape
        d = self.emb_size
        self._exact_catch_up((self.mf_u_embeddings.weight, u_ids), (self.mf_i_embeddings.weight, i_ids),
                             (self.mlp_u_embeddings.weight, u_ids), (self.mlp_i_embeddings.weight, i_ids))
        w_out = self.prediction.weight      # [1, d + last]: GMF part first, MLP part second (NeuMF.py:74)
        # GMF branch: sum_k w[k] * mf_u[b,k] * mf_i[id,k]  == rowdot(w * mf_u[b], mf_i[id])
        mf_u = ops.embedding(self.mf_u_embeddings.weight, u_ids)
        pred = ops.score(ops.colscale(mf_u, w_out[0, :d]), self.mf_i_embeddings.weight, i_ids)
        # MLP tower on [mlp_u[b] ; mlp_i[id]]
        h = ops.gather_concat(self.mlp_u_embeddings.weight, self.mlp_i_embeddings.weight, u_ids, i_ids)
        snap = self._dropout_snapshot(u_ids.device)
        for l, layer in enumerate(self.mlp):
            # relu, then self.dropout_layer (site l of the mask), in the Linear kernel's epilogue
            drop = None if snap is None else ops.Drop(snap, self.dropout_layer.p, l)
            h = ops.linear(h, layer.weight, layer.bias, relu=True, drop=drop)
        pred = pred + ops.linear(h, w_out[:, d:], None, relu=False).view(B, C)
        return {"prediction": pred.view(feed_dict["batch_size"], -1)}

    # test_all without the [Bn * n_items, 2d] concat input: the forward's scores are produced window by window of batch
    # rows by ops.neumf_score_rows, bit for bit, and masked / ranked / selected by the same kernels as the forward's
    # matrix would be, so ranks and lists are the materialised route's.  Outside the envelope (training mode, no clicked
    # sets, a batch below the forward's tensor-core threshold, a layer the forward runs on the SGEMM, a CTA that would not
    # fit) the materialised route runs as before.
    def _all_items_fused(self, feed_dict, clicked, mask_row=None) -> bool:
        if self.training or clicked is None or mask_row is not None or not getattr(self, "test_all", 0):
            return False
        if feed_dict["item_id"].shape[1] != self.item_num:
            return False                    # the materialised route reports the malformed candidate list
        widths = [layer.weight.shape[0] for layer in self.mlp]
        return ops.neumf_all_items_error(self.emb_size, widths, feed_dict["user_id"].numel(), self.item_num) is None

    def _all_items_windows(self, feed_dict):
        """yields (b0, b1, scores [b1 - b0, n_items]) over the batch; the score buffer is reused by the next window"""
        users = feed_dict["user_id"]
        target = feed_dict["item_id"][:, 0]
        Bn = users.numel()
        rows = ops.neumf_window_rows(Bn, self.item_num)
        buf = torch.empty((rows, self.item_num), dtype=torch.float32, device=users.device)
        mlp = [(layer.weight, layer.bias) for layer in self.mlp]
        for b0 in range(0, Bn, rows):
            b1 = min(Bn, b0 + rows)
            yield b0, b1, ops.neumf_score_rows(self.mf_u_embeddings.weight, self.mf_i_embeddings.weight,
                                               self.mlp_u_embeddings.weight, self.mlp_i_embeddings.weight, mlp,
                                               self.prediction.weight, users, target, b0, b1, out=buf[:b1 - b0])

    def eval_ranks(self, feed_dict: dict, mask_row=None, mask_item=None, clicked=None) -> torch.Tensor:
        """_KernelModelMixin.eval_ranks; inside the fused route's envelope only column 0 (the target) of
        feed_dict["item_id"] is read: the other columns must be the test_all list arange(1, n_items), as every
        collate_batch / device_eval_batches batch under test_all has them, since the scorer takes item j for column j."""
        if not self._all_items_fused(feed_dict, clicked, mask_row):
            return super().eval_ranks(feed_dict, mask_row, mask_item, clicked)
        with torch.no_grad():
            self._flush_exact()
            users = feed_dict["user_id"]
            rank = torch.empty(users.numel(), dtype=torch.int64, device=users.device)
            for b0, b1, scores in self._all_items_windows(feed_dict):
                rank[b0:b1] = ops.gt_rank(ops.mask_clicked(scores, users[b0:b1], clicked))
            return rank

    def recommend(self, feed_dict: dict, k: int, clicked=None):
        """_KernelModelMixin.recommend; inside the fused route's envelope only column 0 of feed_dict["item_id"] is
        read, as in eval_ranks"""
        if not self._all_items_fused(feed_dict, clicked):
            return super().recommend(feed_dict, k, clicked)
        with torch.no_grad():
            self._flush_exact()
            users, target = feed_dict["user_id"], feed_dict["item_id"][:, 0]
            kk = min(ops._topk_k(k), self.item_num)
            items = torch.empty((users.numel(), kk), dtype=torch.int64, device=users.device)
            scores = torch.empty((users.numel(), kk), dtype=torch.float32, device=users.device)
            for b0, b1, block in self._all_items_windows(feed_dict):
                cols, vals = ops.topk_rows(ops.mask_clicked(block, users[b0:b1], clicked), k)
                # column 0 is the target, column j >= 1 item j (the candidate list [target | arange(1, n_items)])
                items[b0:b1] = torch.where(cols == 0, target[b0:b1].view(-1, 1), cols)
                scores[b0:b1] = vals
            return items, scores


class _AttentionParams(nn.Module):
    """parameter holder named like utils/layers.py:9-28 (q/k/v Linear with bias, no output projection)"""

    def __init__(self, d):
        super().__init__()
        self.q_linear = nn.Linear(d, d)
        self.k_linear = nn.Linear(d, d)
        self.v_linear = nn.Linear(d, d)


class _TransformerParams(nn.Module):
    """parameter holder named like utils/layers.py:92-110 (post-LN block with d_ff = d)"""

    def __init__(self, d, d_ff):
        super().__init__()
        self.masked_attn_head = _AttentionParams(d)
        self.layer_norm1 = nn.LayerNorm(d)
        self.linear1 = nn.Linear(d, d_ff)
        self.linear2 = nn.Linear(d_ff, d)
        self.layer_norm2 = nn.LayerNorm(d)


class SASRecKernels(_KernelModelMixin):
    """models/sequential/SASRec.py:21-86 (SASRecBase) + utils/layers.py:34-63,112-118 on the library kernels."""

    @staticmethod
    def parse_model_args(parser):
        parser.add_argument("--emb_size", type=int, default=64, help="Size of embedding vectors.")
        parser.add_argument("--num_layers", type=int, default=1, help="Number of self-attention layers.")
        parser.add_argument("--num_heads", type=int, default=4, help="Number of attention heads.")
        parser.add_argument("--table_mode", type=str, default="dense",
                            help="embedding gradient form: dense | sparse | fused (see rechorus_b200.ops)")
        parser.add_argument("--tiled_attention", type=int, default=0,
                            help="1: admit history widths the default attention kernels refuse, on the tiled kernels")
        return parser

    def _base_init(self, args, corpus):
        self.__dict__["_b2r_args"] = args
        self.emb_size = args.emb_size
        self.max_his = args.history_max
        self.num_layers = args.num_layers
        self.num_heads = args.num_heads
        self.tiled_attention = bool(getattr(args, "tiled_attention", 0))
        if self.emb_size % 4 != 0 or self.emb_size % self.num_heads != 0:
            raise ValueError("rechorus_b200 kernels need emb_size % 4 == 0 and emb_size % num_heads == 0")
        if self.max_his > 0:
            # refused here rather than by the first backward (DESIGN.md, a8-a10: the trainable envelope)
            shape = (self.max_his, self.emb_size, self.num_heads, self.num_layers, _SASREC_LASTQ)
            err = ops.seq_train_error(*shape, tiled=self.tiled_attention)
            if err is not None:
                hint = ""
                if not self.tiled_attention and ops.seq_train_error(*shape, tiled=True) is None:
                    hint = "; --tiled_attention 1 runs this shape on the tiled attention kernels"
                raise ValueError(f"SASRec cannot train with history_max={self.max_his}, emb_size={self.emb_size}, "
                                 f"num_heads={self.num_heads}, num_layers={self.num_layers} on these kernels: {err}{hint}")
        ops.check_dropout_p(self.dropout)                    # the reference's nn.Dropout(dropout) (layers.py:104,110)
        self._dropout_init()
        self._base_define_params()
        self.apply(self.init_weights)
        self._register_tables(self.i_embeddings.weight, mode=getattr(args, "table_mode", "dense"))

    def _base_define_params(self):
        # same module names as SASRec.py:41-49 -> identical state_dict keys
        self.i_embeddings = nn.Embedding(self.item_num, self.emb_size)
        self.p_embeddings = nn.Embedding(self.max_his + 1, self.emb_size)
        self.transformer_block = nn.ModuleList(
            [_TransformerParams(self.emb_size, self.emb_size) for _ in range(self.num_layers)])

    def _drops(self, snap, bi):
        if snap is None:
            return None, None
        return ops.Drop(snap, self.dropout, 2 * bi), ops.Drop(snap, self.dropout, 2 * bi + 1)

    def _last_block_one_query(self, blk, x, history, lengths, snap=None, bi=0):
        """The last block for the only position whose output SASRec uses (len-1, SASRec.py:74-81): keys and values from
        every position, query / residual LayerNorms / FFN for that one row per sequence.  Same result as the full block
        followed by select_last, dropout included: the masks are keyed by (sequence, position), not by buffer row."""
        d1, d2 = self._drops(snap, bi)
        Lb = history.shape[1]
        a = blk.masked_attn_head
        ones = torch.ones_like(history)
        x_last = ops.select_last(x, ones, lengths)                               # raw row len-1 (no padding mask yet)
        q_last = ops.linear(x_last, a.q_linear.weight, a.q_linear.bias)
        k = ops.linear(x, a.k_linear.weight, a.k_linear.bias)
        v = ops.linear(x, a.v_linear.weight, a.v_linear.bias)
        ctx_last = ops.attention_last(q_last, k, v, lengths, self.num_heads, tiled=self.tiled_attention)
        c = ops.add_layernorm(ctx_last, x_last, blk.layer_norm1.weight, blk.layer_norm1.bias, drop=d1, lengths=lengths,
                              seq_len=Lb)
        o = ops.linear(ops.linear(c, blk.linear1.weight, blk.linear1.bias, relu=True), blk.linear2.weight, blk.linear2.bias)
        y = ops.add_layernorm(o, c, blk.layer_norm2.weight, blk.layer_norm2.bias, drop=d2, lengths=lengths,
                              seq_len=Lb)  # [B, d]
        t_last = (lengths - 1).clamp(0, history.shape[1] - 1)
        valid = (history.gather(1, t_last.view(-1, 1)) > 0).to(y.dtype)            # SASRec.py:74: y * valid_his
        return y * valid

    def user_state(self, history, lengths, snap=None):
        """snap: the forward's dropout snapshot (None: no dropout)"""
        x = ops.embed_history(self.i_embeddings.weight, self.p_embeddings.weight, history, lengths)   # [B, L, d]
        n_blocks = len(self.transformer_block)
        for bi, blk in enumerate(self.transformer_block):
            if _SASREC_LASTQ and bi == n_blocks - 1:
                return self._last_block_one_query(blk, x, history, lengths, snap, bi)
            d1, d2 = self._drops(snap, bi)
            a = blk.masked_attn_head
            q = ops.linear(x, a.q_linear.weight, a.q_linear.bias)
            k = ops.linear(x, a.k_linear.weight, a.k_linear.bias)
            v = ops.linear(x, a.v_linear.weight, a.v_linear.bias)
            # rows at positions >= len are dead work (the model reads position len-1 only, SASRec.py:74-81, and the
            # mask is causal): skipped exactly
            ctx = ops.causal_attention(q, k, v, self.num_heads, live=lengths, tiled=self.tiled_attention)
            c = ops.add_layernorm(ctx, x, blk.layer_norm1.weight, blk.layer_norm1.bias, drop=d1)       # dropout1 fused
            o = ops.linear(ops.linear(c, blk.linear1.weight, blk.linear1.bias, relu=True),
                           blk.linear2.weight, blk.linear2.bias)
            x = ops.add_layernorm(o, c, blk.layer_norm2.weight, blk.layer_norm2.bias, drop=d2)         # dropout2 fused
        return ops.select_last(x, history, lengths)                                                    # [B, d]

    def query_rows(self, feed_dict):
        with torch.no_grad():
            return self.user_state(feed_dict["history_items"], feed_dict["lengths"]), self.i_embeddings.weight

    def forward(self, feed_dict):
        self.check_list = []
        i_ids = feed_dict["item_id"]            # [B, C]
        history = feed_dict["history_items"]    # [B, Lb] right-padded with 0
        lengths = feed_dict["lengths"]          # [B]
        # history padding (id 0) is never updated by the plan and feeds dead positions only: the flush catches row 0 up
        self._exact_catch_up((self.i_embeddings.weight, history, 0), (self.i_embeddings.weight, i_ids))
        h = self.user_state(history, lengths, self._dropout_snapshot(history.device))
        pred = ops.score(h, self.i_embeddings.weight, i_ids)
        out = {"prediction": pred.view(history.shape[0], -1)}
        if getattr(self, "_b2r_vectors", False):                       # SASRec.py:83-86, kept by SASRecImpression (:121-122)
            out["u_v"] = h.unsqueeze(1).expand(-1, i_ids.shape[1], -1)
            out["i_v"] = ops.embedding(self.i_embeddings.weight, i_ids)
        return out


class ImpressionLossMixin:
    """models/BaseImpressionModel.py:10-128 (ImpressionModel): the list-wise losses over multiple positives / negatives per
    impression, as one kernel family (ops.listwise_loss).  Flags and attribute names are the reference's; the reader and
    runner of the impression setting (ImpressionReader / ImpressionRunner) are the reference's own under the overlay."""

    @staticmethod
    def parse_impression_args(parser):
        parser.add_argument("--loss_n", type=str, default="BPR",
                            help="BPR[hard][after|before] | listnet | softmaxCE | attention_rank (BaseImpressionModel.py:26)")
        parser.add_argument("--train_max_pos_item", type=int, default=20, help="max positive item sample for training")
        parser.add_argument("--train_max_neg_item", type=int, default=20, help="max negative item sample for training")
        parser.add_argument("--test_max_pos_item", type=int, default=20, help="max positive item sample for evaluation")
        parser.add_argument("--test_max_neg_item", type=int, default=20, help="max negative item sample for evaluation")
        return parser

    def _impression_init(self, args):
        self.loss_n = args.loss_n
        self.train_max_pos_item, self.train_max_neg_item = args.train_max_pos_item, args.train_max_neg_item
        self.test_max_pos_item, self.test_max_neg_item = args.test_max_pos_item, args.test_max_neg_item
        ops.listwise_kind(self.loss_n)                    # unknown names fail at construction, not at the first batch
        self.__dict__["_b2r_vectors"] = True

    # BaseImpressionModel.py:44: loss(out_dict, target) -- the ImpressionRunner passes the batch's labels
    def loss(self, out_dict: dict, target=None) -> torch.Tensor:
        if target is None:
            raise ValueError("impression losses need the label tensor (ImpressionRunner passes it as `target`)")
        return ops.listwise_loss(out_dict["prediction"], target, self.loss_n, self.train_max_pos_item)


# ======================================================================================================
# stand-alone hosts mirroring models/BaseModel.py (used when the reference checkout is absent)
# ======================================================================================================


class BaseModel(nn.Module):
    """API mirror of models/BaseModel.py:16-152."""
    reader, runner = None, None
    extra_log_args: List[str] = []

    @staticmethod
    def parse_model_args(parser):
        parser.add_argument("--model_path", type=str, default="", help="Model save path.")
        parser.add_argument("--buffer", type=int, default=1, help="Whether to buffer feed dicts for dev/test")
        return parser

    @staticmethod
    def init_weights(m):
        # BaseModel.py:29-35: N(0, 0.01) for Linear weight AND bias and for Embedding; LayerNorm untouched
        if isinstance(m, nn.Linear):
            nn.init.normal_(m.weight, mean=0.0, std=0.01)
            if m.bias is not None:
                nn.init.normal_(m.bias, mean=0.0, std=0.01)
        elif isinstance(m, nn.Embedding):
            nn.init.normal_(m.weight, mean=0.0, std=0.01)

    def __init__(self, args, corpus):
        super().__init__()
        self.device = args.device
        self.model_path = args.model_path
        self.buffer = args.buffer
        self.optimizer = None
        self.check_list = []

    def forward(self, feed_dict: dict) -> dict:
        raise NotImplementedError

    def loss(self, out_dict: dict) -> torch.Tensor:
        raise NotImplementedError

    def customize_parameters(self) -> list:
        # BaseModel.py:64-73: parameters whose name contains 'bias' get weight_decay 0
        weight_p, bias_p = [], []
        for name, p in self.named_parameters():
            if p.requires_grad:
                (bias_p if "bias" in name else weight_p).append(p)
        return [{"params": weight_p}, {"params": bias_p, "weight_decay": 0}]

    def save_model(self, model_path=None):
        opt = self.__dict__.get("_b2r_optimizer")
        if getattr(opt, "exact_dense", False):
            opt.flush()                     # the checkpoint holds dense-Adam weights in either train or eval mode
        model_path = model_path or self.model_path
        d = os.path.dirname(model_path)
        if d:
            os.makedirs(d, exist_ok=True)
        torch.save(self.state_dict(), model_path)

    def load_model(self, model_path=None):
        model_path = model_path or self.model_path
        self.load_state_dict(torch.load(model_path, map_location=self.device))
        logging.info("Load model from " + model_path)

    def count_variables(self) -> int:
        return sum(p.numel() for p in self.parameters() if p.requires_grad)

    def actions_after_train(self):
        pass

    class Dataset(TorchDataset):
        """BaseModel.py:98-152: per-phase view of the corpus that yields feed dicts and collates them."""

        def __init__(self, model, corpus, phase: str):
            self.model, self.corpus, self.phase = model, corpus, phase
            self.buffer_dict = {}
            self.data = corpus.data_df[phase].to_dict("list")

        def __len__(self):
            for key in self.data:
                return len(self.data[key])
            return 0

        def __getitem__(self, index: int) -> dict:
            if self.model.buffer and self.phase != "train":
                return self.buffer_dict[index]
            return self._get_feed_dict(index)

        def _get_feed_dict(self, index: int) -> dict:
            raise NotImplementedError

        def prepare(self):
            if self.model.buffer and self.phase != "train":
                for i in range(len(self)):
                    self.buffer_dict[i] = self._get_feed_dict(i)

        def actions_before_epoch(self):
            pass

        def collate_batch(self, feed_dicts: List[dict]) -> dict:
            # BaseModel.py:135-152: stack equal-length arrays; right-pad ragged ones (histories) with 0
            out = {}
            for key in feed_dicts[0]:
                vals = [d[key] for d in feed_dicts]
                ragged = isinstance(vals[0], np.ndarray) and any(len(v) != len(vals[0]) for v in vals)
                if ragged:
                    out[key] = pad_sequence([torch.from_numpy(np.asarray(v)) for v in vals], batch_first=True)
                else:
                    out[key] = torch.from_numpy(np.array(vals))
            out["batch_size"] = len(feed_dicts)
            out["phase"] = self.phase
            return out


class GeneralModel(BaseModel):
    """API mirror of models/BaseModel.py:154-214."""
    reader, runner = "BaseReader", "BaseRunner"

    @staticmethod
    def parse_model_args(parser):
        parser.add_argument("--num_neg", type=int, default=1, help="The number of negative items during training.")
        parser.add_argument("--dropout", type=float, default=0, help="Dropout probability for each deep layer")
        parser.add_argument("--test_all", type=int, default=0, help="Whether testing on all the items.")
        return BaseModel.parse_model_args(parser)

    def __init__(self, args, corpus):
        super().__init__(args, corpus)
        self.user_num = corpus.n_users
        self.item_num = corpus.n_items
        self.num_neg = args.num_neg
        self.dropout = args.dropout
        self.test_all = args.test_all

    class Dataset(BaseModel.Dataset):
        def _get_feed_dict(self, index):
            # BaseModel.py:192-203: column 0 = target, then the negatives (all items when test_all)
            target = self.data["item_id"][index]
            if self.phase != "train" and self.model.test_all:
                negs = np.arange(1, self.corpus.n_items)
            else:
                negs = self.data["neg_items"][index]
            return {"user_id": self.data["user_id"][index],
                    "item_id": np.concatenate([[target], negs]).astype(int)}

        def actions_before_epoch(self):
            sampler = self.model.__dict__.get("_b2r_device_sampler")
            if sampler is not None:
                # opt-in (runner --device_sampler 1; row f3 groundwork): same distribution drawn on the GPU from a
                # counter-based stream keyed by (seed, epoch) instead of the Python rejection loop below
                epoch = self.__dict__.get("_b2r_epoch", 0) + 1
                self.__dict__["_b2r_epoch"] = epoch
                users = torch.as_tensor(np.asarray(self.data["user_id"], dtype=np.int64)).to(self.model.device)
                self.data["neg_items"] = sampler.sample(users, self.model.num_neg, epoch).cpu().numpy()
                return
            # BaseModel.py:206-214: uniform negatives from NumPy's global RNG, rejected against train clicks
            n = len(self)
            neg = np.random.randint(1, self.corpus.n_items, size=(n, self.model.num_neg))
            clicked = self.corpus.train_clicked_set
            for i, u in enumerate(self.data["user_id"]):
                seen = clicked[u]
                for j in range(self.model.num_neg):
                    while neg[i][j] in seen:
                        neg[i][j] = np.random.randint(1, self.corpus.n_items)
            self.data["neg_items"] = neg


class SequentialModel(GeneralModel):
    """API mirror of models/BaseModel.py:216-245."""
    reader = "SeqReader"

    @staticmethod
    def parse_model_args(parser):
        parser.add_argument("--history_max", type=int, default=20, help="Maximum length of history.")
        return GeneralModel.parse_model_args(parser)

    def __init__(self, args, corpus):
        super().__init__(args, corpus)
        self.history_max = args.history_max

    class Dataset(GeneralModel.Dataset):
        def __init__(self, model, corpus, phase):
            super().__init__(model, corpus, phase)
            keep = np.array(self.data["position"]) > 0          # history length must be non-zero
            for key in self.data:
                self.data[key] = np.array(self.data[key], dtype=object)[keep].tolist()

        def _get_feed_dict(self, index):
            fd = super()._get_feed_dict(index)
            pos = self.data["position"][index]
            seq = self.corpus.user_his[fd["user_id"]][:pos]
            if self.model.history_max > 0:
                seq = seq[-self.model.history_max:]
            fd["history_items"] = np.array([x[0] for x in seq])
            fd["history_times"] = np.array([x[1] for x in seq])
            fd["lengths"] = len(fd["history_items"])
            return fd


# ======================================================================================================
# concrete stand-alone models
# ======================================================================================================


class BPRMF(BPRMFKernels, GeneralModel):
    """Drop-in for models/general/BPRMF.py:47-63."""
    reader, runner = "BaseReader", "BaseRunner"
    extra_log_args = ["emb_size", "batch_size"]

    @staticmethod
    def parse_model_args(parser):
        parser = BPRMFKernels.parse_model_args(parser)
        return GeneralModel.parse_model_args(parser)

    def __init__(self, args, corpus):
        GeneralModel.__init__(self, args, corpus)
        self._base_init(args, corpus)


class NeuMF(NeuMFKernels, GeneralModel):
    """Drop-in for models/general/NeuMF.py:22-76."""
    reader, runner = "BaseReader", "BaseRunner"
    extra_log_args = ["emb_size", "layers"]

    @staticmethod
    def parse_model_args(parser):
        parser = NeuMFKernels.parse_model_args(parser)
        return GeneralModel.parse_model_args(parser)

    def __init__(self, args, corpus):
        GeneralModel.__init__(self, args, corpus)
        self._neumf_init(args, corpus)


class SASRec(SASRecKernels, SequentialModel):
    """Drop-in for models/sequential/SASRec.py:89-105."""
    reader, runner = "SeqReader", "BaseRunner"
    extra_log_args = ["emb_size", "num_layers", "num_heads"]

    @staticmethod
    def parse_model_args(parser):
        parser = SASRecKernels.parse_model_args(parser)
        return SequentialModel.parse_model_args(parser)

    def __init__(self, args, corpus):
        SequentialModel.__init__(self, args, corpus)
        self._base_init(args, corpus)


class BPRMFImpression(ImpressionLossMixin, BPRMFKernels, GeneralModel):
    """Drop-in for models/general/BPRMF.py:65-80 (stand-alone form: bring your own impression batches)."""
    reader, runner = "ImpressionReader", "ImpressionRunner"
    extra_log_args = ["emb_size", "batch_size"]

    @staticmethod
    def parse_model_args(parser):
        parser = BPRMFKernels.parse_model_args(parser)
        parser = ImpressionLossMixin.parse_impression_args(parser)
        return GeneralModel.parse_model_args(parser)

    def __init__(self, args, corpus):
        GeneralModel.__init__(self, args, corpus)
        self._impression_init(args)
        self._base_init(args, corpus)


class SASRecImpression(ImpressionLossMixin, SASRecKernels, SequentialModel):
    """Drop-in for models/sequential/SASRec.py:107-122."""
    reader, runner = "ImpressionSeqReader", "ImpressionRunner"
    extra_log_args = ["emb_size", "num_layers", "num_heads"]

    @staticmethod
    def parse_model_args(parser):
        parser = SASRecKernels.parse_model_args(parser)
        parser = ImpressionLossMixin.parse_impression_args(parser)
        return SequentialModel.parse_model_args(parser)

    def __init__(self, args, corpus):
        SequentialModel.__init__(self, args, corpus)
        self._impression_init(args)
        self._base_init(args, corpus)
