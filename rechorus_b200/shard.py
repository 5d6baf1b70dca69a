"""Row-range sharded BPRMF tables across the GPUs of one box (BASELINE config 5) -- *score routing*.

The reference is single-device (SURVEY.md section 2.1: no collectives anywhere); this module is new.  It applies
only where a table does not fit one GPU with its optimizer state (100 M x 128 fp32 + Adam = 154 GB); configs 1-4
are replicas-only and never come here.

Per step every rank holds a local batch (user_id [B], item_id [B, C], GLOBAL ids) and owns rows
``[rank*rows, (rank+1)*rows)`` of each table.  One exchange per direction, NCCL all-to-all over NVLink:

  fwd  user ids -> owners, user vectors back (B x d, small)            all_to_all x2
       all-gather of the B user vectors (W*B x d, a few MB)            all_gather
       (sample, local row) pairs bucketed by owner                     all_to_all
       owners score their pairs against the gathered user vectors
       (b2r_pairdot_fwd) and return 4-byte scores                      all_to_all
  bwd  home: BPR loss + gradient g; g -> owners                        all_to_all
       owners: dQ partials (bucketed dense add) and the fused row-sparse optimizer on their item shard
       reduce-scatter of the dQ partials to the home ranks             reduce_scatter
       dQ rows -> user-row owners, fused optimizer on the user shard   all_to_all

Routing 4-byte scores instead of 4d-byte rows keeps the exchange at ~30 MB per rank per step at config-5 sizes
(vector routing would move ~1 GB and be NVLink-bound, SURVEY.md section 8e), so the step stays HBM-bound on the
owners' gather / optimizer kernels.  Exchange buffers have a fixed per-destination capacity
(``cap_factor`` x the uniform share) so that no host synchronisation is needed to size them; a batch whose ids
overflow a destination trips a device-side assert.

The global objective is the mean BPR loss over the W*B samples of the step (each rank's local mean / W).

All arithmetic goes through a *backend*: ``CudaBackend`` (the sm_90a kernels; the product) -- the tests inject a
CPU stand-in to exercise the exchange bookkeeping under gloo.

Two forms of the exchange:
  * ``exchange="p2p"`` (default on CUDA): every hop above is done BY THE KERNELS over peer-mapped symmetric memory
    (csrc/shard_p2p.cu, csrc/pairdot_p2p.cu): the routing kernel stores each pair straight into its owner's receive
    arrays, owners store user vectors into every rank's block and scores into the requester's buffer, g and the dQ rows
    travel the same way, and the dQ partials are summed from peer memory in rank order.  Six signal-pad barriers order
    the phases; there is no NCCL call and no tensor glue on the data path.
  * ``exchange="nccl"``: the collective form described above (the baseline; also what the gloo tests exercise).
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.distributed as dist


class CudaBackend:
    """local compute on the library kernels (rechorus_b200.ops); no CPU fallback"""

    def gather_rows(self, T, ids):
        from . import ops
        return ops.gather_rows(T, ids)

    def pairdot(self, Q, qidx, T, rows):
        from . import ops
        return ops.pairdot(Q, qidx, T, rows)

    def pairdot_p2p(self, Q, qidx, T, rows, out_tab, seg):
        from . import ops
        ops.pairdot_p2p(Q, qidx, T, rows, out_tab, seg)

    def bpr_loss_and_grad(self, pred):
        from . import ops
        return ops.bpr_loss_and_grad(pred)

    def sum_runs(self, out, key, rows, coef, T):
        """out[key[e]] = sum over each contiguous run of valid (rows >= 0) pairs with that key of coef[e] * T[rows[e]]"""
        from . import ops
        ops.pair_runs_sum(out, key, rows, coef, T)

    def optimizer_rows(self, W, state, ids, src, coef, src_id, opt):
        """row-sparse optimizer on W for the rows ids[p] >= 0 with gradient sum_p coef[p] * src[src_id[p]]"""
        from . import ops
        n = ids.numel()
        plan = ops.make_plan(ids, W.shape[0], W.shape[1], ignore_id=-1, ignore_n=n)
        plan.apply_optimizer(W, state.get("m"), state.get("v"), opt, [ops.Source(src=src, n=n, coef=coef, src_id=src_id)])

    def make_opt(self, name, lr, betas, eps, wd, t):
        from . import lib
        kind = {"SGD": lib.OPT_SGD, "Adam": lib.OPT_ADAM, "Adagrad": lib.OPT_ADAGRAD}[name]
        return lib.Optim(kind, lr, betas[0], betas[1], eps, wd, 1.0 - betas[0] ** t, 1.0 - betas[1] ** t, 0)


def _bucket_by_owner(owner: torch.Tensor, world: int):
    """stable partition of positions by owner: returns (order, owner_sorted, rank_within_owner, counts)"""
    if world == 1:
        n = owner.numel()
        ar = torch.arange(n, device=owner.device)
        return ar, torch.zeros_like(owner), ar, torch.full((1,), n, dtype=torch.int64, device=owner.device)
    # 8-bit keys: one radix pass instead of eight (W <= 255 ranks on one box)
    key_sorted, order = torch.sort(owner.to(torch.uint8), stable=True)
    owner_sorted = key_sorted.to(torch.int64)
    # segment starts by binary search in the sorted keys (a histogram of 1 M values into <= 8 bins is all atomics)
    bounds = torch.searchsorted(key_sorted, torch.arange(world + 1, device=owner.device, dtype=torch.uint8).clamp(max=255)
                                if world < 255 else torch.arange(world + 1, device=owner.device), right=False)
    bounds[-1] = owner.numel()
    starts = bounds[:-1]
    counts = bounds[1:] - bounds[:-1]
    rank = torch.arange(owner.numel(), device=owner.device) - starts[owner_sorted]
    return order, owner_sorted, rank, counts


class ShardedBPRMF:
    def __init__(self, n_users: int, n_items: int, d: int, device, backend=None, group=None, optimizer: str = "Adam",
                 lr: float = 1e-3, l2: float = 0.0, betas=(0.9, 0.999), eps: Optional[float] = None,
                 cap_factor: float = 1.25, seed: int = 0, init_std: float = 0.01, world_override: Optional[int] = None,
                 exchange: Optional[str] = None):
        """world_override=1: hold the WHOLE table on this rank and exchange nothing even inside an initialised process
        group (the 1-GPU anchor of the scaling curve, run by one rank while the others wait).
        exchange: "p2p" or "nccl" (module docstring); None picks "p2p" on CUDA without an injected backend, else
        "nccl".  "p2p" runs the library kernels on CUDA memory, so it needs both."""
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if world_override is not None:
            if world_override != 1:
                raise ValueError("world_override can only force the single-rank form")
            self.world, self.rank = 1, 0
        self.n_users, self.n_items, self.d, self.device = n_users, n_items, d, device
        self.rows_u = math.ceil(n_users / self.world)
        self.rows_i = math.ceil(n_items / self.world)
        self.backend = backend or CudaBackend()
        self.opt_name, self.lr, self.l2, self.betas = optimizer, lr, l2, betas
        self.eps = {"SGD": 0.0, "Adam": 1e-8, "Adagrad": 1e-10}[optimizer] if eps is None else eps
        self.cap_factor = cap_factor
        self.t = 0
        p2p_ok = torch.device(device).type == "cuda" and backend is None
        if exchange is None:
            exchange = "p2p" if p2p_ok else "nccl"
        elif exchange not in ("p2p", "nccl"):
            raise ValueError(f"exchange must be 'p2p' or 'nccl', got {exchange!r}")
        elif exchange == "p2p" and not p2p_ok:
            raise ValueError("exchange='p2p' needs a CUDA device and the library backend")
        self.exchange = exchange
        self._p2p = None
        g = torch.Generator(device=device).manual_seed(seed * 1000 + self.rank)
        # models/BaseModel.py:29-35 init, one shard per rank
        self.U = torch.empty(self.rows_u, d, device=device).normal_(0.0, init_std, generator=g)
        self.I = torch.empty(self.rows_i, d, device=device).normal_(0.0, init_std, generator=g)
        self.state_u, self.state_i = {}, {}
        for st, W in ((self.state_u, self.U), (self.state_i, self.I)):
            if optimizer == "Adam":
                st["m"] = torch.zeros_like(W)
            if optimizer != "SGD":
                st["v"] = torch.zeros_like(W)

    # -- collectives (degenerate to copies for a single rank) --------------------------------------------
    def _a2a(self, x: torch.Tensor) -> torch.Tensor:
        if self.world == 1:
            return x.clone()
        out = torch.empty_like(x)
        dist.all_to_all_single(out, x.contiguous(), group=self.group)
        return out

    def _all_gather(self, x: torch.Tensor) -> torch.Tensor:
        if self.world == 1:
            return x.clone()
        out = torch.empty((self.world * x.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(out, x.contiguous(), group=self.group)
        return out

    def _reduce_scatter(self, x: torch.Tensor) -> torch.Tensor:
        if self.world == 1:
            return x.clone()
        out = torch.empty((x.shape[0] // self.world,) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        dist.reduce_scatter_tensor(out, x.contiguous(), op=dist.ReduceOp.SUM, group=self.group)
        return out

    def exchange_description(self) -> str:
        if self.world == 1:
            return "none (single rank)"
        if self.exchange == "p2p":
            return ("score routing, fused into the kernels: pairs / user vectors / scores / g / dQ rows stored into the peers' "
                    "symmetric-memory buffers by the producing kernels, dQ partials summed from peer memory in rank order; "
                    "6 signal-pad barriers per step, no NCCL collective on the data path")
        return "score routing over NCCL: all-to-all x6, all-gather, reduce-scatter per step"

    def nvlink_bytes_per_step(self, B: int, C: int) -> int:
        """bytes this rank sends to peers per step (the (W-1)/W remote share of every hop)"""
        W, d = self.world, self.d
        if W == 1:
            return 0
        cap = self.capacity(B * C)
        per_dest = (B * 8 + B * d * 4                       # user ids out, user vectors back
                    + cap * 8 + cap * 4 + cap * 4            # pairs out, scores back, g out
                    + B * d * 4                              # dQ rows to the user-row owners
                    + B * d * 4)                             # reduce-scatter share of the dQ partials
        return int((W - 1) * (per_dest + B * d * 4))         # + all-gather of the user vectors

    def capacity(self, n: int) -> int:
        if self.world == 1:
            return n
        return min(n, int(math.ceil(n / self.world * self.cap_factor)) + 64)

    # -- one training step ----------------------------------------------------------------------------
    def scores(self, uid: torch.Tensor, iid: torch.Tensor):
        """forward only: returns (pred [B,C], routing state for the backward)"""
        W, B, d, be = self.world, uid.numel(), self.d, self.backend
        C = iid.shape[1]
        n = B * C
        dev = uid.device
        # A. user vectors from their owners
        own_u = torch.div(uid, self.rows_u, rounding_mode="floor")
        ord_u, own_us, rank_u, _ = _bucket_by_owner(own_u, W)
        send_uid = torch.full((W, B), -1, dtype=torch.int64, device=dev)
        send_uid[own_us, rank_u] = (uid - own_u * self.rows_u)[ord_u]
        recv_uid = self._a2a(send_uid)                                           # [W(src), B] local rows or -1
        vec_recv = self._a2a(be.gather_rows(self.U, recv_uid.clamp(min=0)))       # [W(owner), B, d]
        slot_u = torch.empty(B, dtype=torch.int64, device=dev)
        slot_u[ord_u] = own_us * B + rank_u                                       # where sample b's vector landed
        q = be.gather_rows(vec_recv.view(W * B, d), slot_u)                       # [B, d]
        # B. every owner needs every sample's user vector
        q_all = self._all_gather(q)                                               # [W*B, d], row = src*B + b
        # C. (sample, local row) pairs to the item-row owners, fixed capacity per destination
        flat = iid.reshape(-1)
        own_i = torch.div(flat, self.rows_i, rounding_mode="floor")
        ord_i, own_is, rank_i, counts_i = _bucket_by_owner(own_i, W)
        cap = self.capacity(n)
        torch._assert_async(counts_i.max() <= cap)                                # ids too skewed for cap_factor
        if B >= (1 << 21):
            raise ValueError("per-rank batch too large for the packed (row, sample) exchange format")
        send_pairs = torch.full((W, cap), -1, dtype=torch.int64, device=dev)      # (local row << 21) | sample index
        keep_rank = rank_i.clamp(max=cap - 1)
        send_pairs[own_is, keep_rank] = ((flat - own_i * self.rows_i)[ord_i] << 21) | torch.div(ord_i, C, rounding_mode="floor")
        recv_pairs = self._a2a(send_pairs)                                        # [W(src), cap]
        rows = recv_pairs >> 21                                                   # -1 stays -1 (arithmetic shift)
        src_base = (torch.arange(W, device=dev) * B).view(W, 1)
        qidx = (recv_pairs & ((1 << 21) - 1)) + src_base                          # row of q_all (garbage where rows < 0)
        qidx = torch.where(rows >= 0, qidx, torch.zeros_like(qidx))
        # D. owners score, scores travel back
        sc_recv = self._a2a(be.pairdot(q_all, qidx, self.I, rows).view(W, cap))   # [W(owner), cap]
        pred = torch.empty(n, dtype=torch.float32, device=dev)
        pred[ord_i] = sc_recv[own_is, keep_rank]
        state = dict(B=B, C=C, n=n, cap=cap, ord_u=ord_u, own_us=own_us, rank_u=rank_u, recv_uid=recv_uid,
                     ord_i=ord_i, own_is=own_is, keep_rank=keep_rank, rows=rows, qidx=qidx, q_all=q_all)
        return pred.view(B, C), state

    def train_step(self, uid: torch.Tensor, iid: torch.Tensor) -> torch.Tensor:
        if self.exchange == "p2p":
            return self._train_step_p2p(uid, iid)
        W, d, be = self.world, self.d, self.backend
        pred, st = self.scores(uid, iid)
        B, C, cap = st["B"], st["C"], st["cap"]
        dev = uid.device
        # E. local loss; the step's objective is the mean over the W*B global samples
        loss, g = be.bpr_loss_and_grad(pred)
        g = g / W
        # F. g to the owners, in the order the pairs were sent
        g_send = torch.zeros((W, cap), dtype=torch.float32, device=dev)
        g_send[st["own_is"], st["keep_rank"]] = g.reshape(-1)[st["ord_i"]]
        g_recv = self._a2a(g_send).reshape(-1)                                    # [W*cap], 0 in unused slots
        rows, qidx, q_all = st["rows"].reshape(-1), st["qidx"].reshape(-1), st["q_all"]
        self.t += 1
        opt_i = be.make_opt(self.opt_name, self.lr, self.betas, self.eps, self.l2, self.t)
        # G. dQ partials for every (src, sample) this owner served: dQ[src*B+b] += g * I[row]   (before I moves)
        dq_part = torch.zeros((W * B, d), dtype=torch.float32, device=dev)
        be.sum_runs(dq_part, qidx, rows, g_recv, self.I)
        # H. item shard: fused row-sparse optimizer, gradient row = sum g * q_all[qidx]
        be.optimizer_rows(self.I, self.state_i, rows, q_all, g_recv, qidx, opt_i)
        # I. home ranks get their samples' dQ summed over the owners
        dq = self._reduce_scatter(dq_part)                                        # [B, d]
        # J. dQ rows to the user-row owners, fused optimizer on the user shard
        dq_send = torch.zeros((W, B, d), dtype=torch.float32, device=dev)
        dq_send[st["own_us"], st["rank_u"]] = dq[st["ord_u"]]
        dq_recv = self._a2a(dq_send).view(W * B, d)
        recv_uid = st["recv_uid"].reshape(-1)
        ar = torch.arange(W * B, device=dev)
        be.optimizer_rows(self.U, self.state_u, recv_uid, dq_recv, torch.ones(W * B, dtype=torch.float32, device=dev),
                          ar, opt_i)
        return loss

    # ---------------------------------------------------------------------------------------------------------------
    # exchange="p2p": the same step with every hop done by kernels over peer-mapped symmetric memory
    # ---------------------------------------------------------------------------------------------------------------
    def _p2p_setup(self, B: int, C: int):
        import ctypes as Ct
        from . import lib as _lib
        W, d, dev = self.world, self.d, self.U.device
        n = B * C
        cap = self.capacity(n)
        L = _lib.load()
        lay, off = {}, 0

        def take(name, nbytes):
            nonlocal off
            lay[name] = off
            off += (nbytes + 255) // 256 * 256

        take("rows_in", W * cap * 8)
        take("qidx_in", W * cap * 8)
        take("scores_in", W * cap * 4)
        take("g_in", W * cap * 4)
        for par in (0, 1):                      # written by the NEXT step's routing while this step's user update reads
            take(f"ureq_rows{par}", W * B * 8)
            take(f"ureq_q{par}", W * B * 8)
        take("q_all", W * B * d * 4)
        take("dqp", W * B * d * 4)
        take("dqu_in", W * B * d * 4)
        total = off
        if W > 1:
            import torch.distributed._symmetric_memory as symm
            buf = symm.empty(total, dtype=torch.uint8, device=dev)
            hdl = symm.rendezvous(buf, self.group if self.group is not None else dist.group.WORLD)
            bases = [int(hdl.buffer_ptrs[r]) for r in range(W)]
        else:
            buf, hdl = torch.empty(total, dtype=torch.uint8, device=dev), None
            bases = [buf.data_ptr()]
        buf.zero_()

        def view(name, dtype, shape):
            nb = torch.empty((), dtype=dtype).element_size()
            cnt = 1
            for x in shape:
                cnt *= x
            return buf[lay[name]:lay[name] + cnt * nb].view(dtype).view(*shape)

        def table(name, region_bytes=0):
            """host array of W device pointers: rank r's buffer `name` (+ this rank's region inside it)"""
            return (Ct.c_void_p * W)(*[bases[r] + lay[name] + self.rank * region_bytes for r in range(W)])

        x = types_ns = type("P2P", (), {})()
        x.B, x.C, x.n, x.cap, x.hdl, x.buf = B, C, n, cap, hdl, buf
        x.rows_in, x.qidx_in = view("rows_in", torch.int64, (W * cap,)), view("qidx_in", torch.int64, (W * cap,))
        x.scores_in, x.g_in = view("scores_in", torch.float32, (W * cap,)), view("g_in", torch.float32, (W * cap,))
        x.ureq_rows = [view(f"ureq_rows{p}", torch.int64, (W * B,)) for p in (0, 1)]
        x.ureq_q = [view(f"ureq_q{p}", torch.int64, (W * B,)) for p in (0, 1)]
        x.q_all, x.dqp = view("q_all", torch.float32, (W * B, d)), view("dqp", torch.float32, (W * B, d))
        x.dqu_in = view("dqu_in", torch.float32, (W * B, d))
        # where this rank writes at each peer
        x.t_rows, x.t_qidx = table("rows_in", cap * 8), table("qidx_in", cap * 8)
        x.t_g = table("g_in", cap * 4)
        x.t_ureq_rows = [table(f"ureq_rows{p}", B * 8) for p in (0, 1)]
        x.t_ureq_q = [table(f"ureq_q{p}", B * 8) for p in (0, 1)]
        x.t_q_all, x.t_dqp = table("q_all"), table("dqp")
        x.t_dqu = table("dqu_in", B * d * 4)
        x.score_tab = torch.tensor([bases[r] + lay["scores_in"] + self.rank * cap * 4 for r in range(W)], dtype=torch.int64,
                                   device=dev)
        # local scratch
        x.slot_of = torch.empty(n, dtype=torch.int32, device=dev)
        x.slot_of_u = torch.empty(B, dtype=torch.int32, device=dev)
        x.tot = torch.zeros(2 * W, dtype=torch.int32, device=dev)
        x.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        x.route_ws = torch.empty(L.b2r_route_workspace_bytes(B, W), dtype=torch.uint8, device=dev)
        x.dq = torch.empty((B, d), dtype=torch.float32, device=dev)
        x.ones = torch.ones(W * B, dtype=torch.float32, device=dev)
        x.arange = torch.arange(W * B, dtype=torch.int64, device=dev)
        x.step = 0
        if hdl is not None:
            hdl.barrier(channel=0)              # every rank's buffers are zeroed before anyone writes into them
        return x

    def _barrier(self, x, ch: int):
        if x.hdl is not None:
            x.hdl.barrier(channel=ch)

    def _train_step_p2p(self, uid: torch.Tensor, iid: torch.Tensor) -> torch.Tensor:
        from . import lib as _lib, ops
        W, d, be, me = self.world, self.d, self.backend, self.rank
        B, C = iid.shape
        x = self._p2p
        if x is None or x.B != B or x.C != C:
            x = self._p2p = self._p2p_setup(B, C)
        L = _lib.load()
        st = torch.cuda.current_stream().cuda_stream
        ef = ops.err_flag(uid.device).data_ptr()
        uid, iid = uid.contiguous(), iid.contiguous()
        par = x.step & 1
        x.step += 1
        # 0. route: pairs and user-row requests land in their owners' receive arrays (peer stores from the kernel)
        _lib.check(L.b2r_route_ids(iid.data_ptr(), B, C, W, self.rows_i, self.n_items, x.t_rows, x.t_qidx, me * B, x.cap,
                                   x.slot_of.data_ptr(), x.tot.data_ptr(), x.overflow.data_ptr(), x.route_ws.data_ptr(),
                                   x.route_ws.numel(), ef, st), "b2r_route_ids(items)")
        _lib.check(L.b2r_route_ids(uid.data_ptr(), B, 1, W, self.rows_u, self.n_users, x.t_ureq_rows[par], x.t_ureq_q[par],
                                   me * B, B, x.slot_of_u.data_ptr(), x.tot.data_ptr() + 4 * W, x.overflow.data_ptr(),
                                   x.route_ws.data_ptr(), x.route_ws.numel(), ef, st), "b2r_route_ids(users)")
        torch._assert_async(x.overflow[0] == 0)               # ids too skewed for cap_factor
        self._barrier(x, 0)
        # 1. owners of user rows fill every rank's block of user vectors (gather + all-gather in one kernel)
        _lib.check(L.b2r_serve_rows(self.U.data_ptr(), self.U.shape[0], x.ureq_rows[par].data_ptr(), x.ureq_q[par].data_ptr(),
                                    W * B, x.t_q_all, W, d, ef, st), "b2r_serve_rows")
        self._barrier(x, 1)
        # 2. owners score their pairs; each score is stored into the requester's buffer by the scoring kernel
        be.pairdot_p2p(x.q_all, x.qidx_in, self.I, x.rows_in, x.score_tab, x.cap)
        self._barrier(x, 2)
        # 3. home: scores -> [B, C], BPR loss + gradient (objective = mean over the W*B samples), g -> owners
        pred = x.scores_in[x.slot_of.long()].view(B, C)
        loss, g = be.bpr_loss_and_grad(pred)
        _lib.check(L.b2r_scatter_f32_to_peers(g.data_ptr(), x.slot_of.data_ptr(), x.n, x.t_g, W, x.cap, 1.0 / W, st),
                   "b2r_scatter_f32_to_peers")
        self._barrier(x, 3)
        # 4. owners: dQ partials per (source, sample), then the fused row-sparse optimizer on the item shard
        self.t += 1
        opt = be.make_opt(self.opt_name, self.lr, self.betas, self.eps, self.l2, self.t)
        x.dqp.zero_()
        be.sum_runs(x.dqp, x.qidx_in, x.rows_in, x.g_in, self.I)
        be.optimizer_rows(self.I, self.state_i, x.rows_in, x.q_all, x.g_in, x.qidx_in, opt)
        self._barrier(x, 4)
        # 5. home: dQ = sum of the owners' partials read from peer memory in rank order; rows -> user-row owners
        _lib.check(L.b2r_sum_rows_from_peers(x.t_dqp, W, me * B * d, x.dq.data_ptr(), B * d, st), "b2r_sum_rows_from_peers")
        _lib.check(L.b2r_scatter_rows_to_peers(x.dq.data_ptr(), x.slot_of_u.data_ptr(), B, x.t_dqu, W, B, d, st),
                   "b2r_scatter_rows_to_peers")
        self._barrier(x, 5)
        # 6. owners: fused row-sparse optimizer on the user shard
        be.optimizer_rows(self.U, self.state_u, x.ureq_rows[par], x.dqu_in, x.ones, x.arange, opt)
        return loss
