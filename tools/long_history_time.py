#!/usr/bin/env python
"""SASRec attention and training steps at long histories (--tiled_attention), in one process, with the card's name, power
limit and max SM clock read in the same run.  One JSON line per measurement.

  (a) tiled vs register-resident causal attention, forward + backward, at bench.py c4's d = 64, H = 4, B = 4096 and
      L in {50, 128} (inside the rt kernels' envelope), alternating the two in the timed loop; the bits must be equal
  (b) tiled forward + backward at L in {200, 512, 1024}, d/H in {16, 64} (d = 64), B * L = 262144 rows: achieved FP32
      FLOP/s from the FLOPs causal attention needs (computed from the shapes below) against the H100 SXM data sheet's
      67 TFLOP/s
  (c) one whole SASRec training step (fused Adam) replayed as a CUDA graph, B = 4096, K = 99 negatives, d = 64, H = 4:
      history_max 200 with 2 blocks, and 512 with 1 block; against an eager stock-PyTorch fp32 SASRec step written here
      (nn.Linear, the masked softmax of utils/layers.py, nn.LayerNorm, torch.optim.Adam) on the same GPU and weights.
      The losses on the same weights and after the 2nd and 3rd updates are printed for both and must agree to 1e-5.

    python tools/long_history_time.py [--iters 20]

Attention FLOPs: a causal row i meets keys 0..i, so a sequence has T = L (L + 1) / 2 (query, key) pairs per head.  The
forward needs QK^T and PV (2 matmuls), the backward QK^T again, dO V^T, dS K, dS^T Q and P^T dO (5): each matmul costs
2 dk FLOP per pair, so fwd + bwd = 14 * B * H * T * dk.  Exponentials and the softmax bookkeeping are not counted.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import types

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_PEAK = 67e12           # H100 SXM data sheet, dense FP32, 700 W card


def card():
    dev = torch.device("cuda", 0)
    out = {"gpu": torch.cuda.get_device_name(dev)}
    q = subprocess.run(["nvidia-smi", "-i", str(dev.index), "--query-gpu=power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
    pl, clk = [x.strip() for x in q.strip().splitlines()[0].split(",")]
    out["power_limit_w"], out["sm_max_mhz"] = float(pl), int(float(clk))
    return out


def emit(**kw):
    print(json.dumps(kw), flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# (a), (b): attention through the C ABI
# ---------------------------------------------------------------------------------------------------------------------

class Attn:
    """fwd + bwd of one kind (rt | tiled) with preallocated outputs, so the timed loop only launches"""

    def __init__(self, kind, q, k, v, live, go, H):
        from rechorus_b200 import lib as L
        self.h, self.kind, self.H = L.load(), kind, H
        B, Ln, d = q.shape
        self.shape = (B, Ln, d)
        self.q, self.k, self.v, self.live, self.go = q, k, v, live, go
        self.ctx, self.lse = torch.empty_like(q), torch.empty(B, Ln, H, device=q.device)
        self.dq, self.dk, self.dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
        self.ws = torch.empty(int(self.h.b2r_attention_bwd_tiled_workspace_bytes(B, Ln, H)), dtype=torch.uint8,
                              device=q.device)

    def __call__(self):
        from rechorus_b200 import lib as L
        B, Ln, d = self.shape
        p = lambda t: t.data_ptr()                          # noqa: E731
        L.check(getattr(self.h, f"b2r_attention_fwd_{self.kind}")(p(self.q), p(self.k), p(self.v), d, p(self.live),
                                                                  p(self.ctx), p(self.lse), B, Ln, d, self.H, 0), "fwd")
        args = [p(self.q), p(self.k), p(self.v), d, p(self.live), p(self.ctx), p(self.lse), p(self.go), p(self.dq),
                p(self.dk), p(self.dv), d, B, Ln, d, self.H]
        if self.kind == "tiled":
            args += [p(self.ws), self.ws.numel()]
        L.check(getattr(self.h, f"b2r_attention_bwd_{self.kind}")(*args, 0), "bwd")

    def results(self):
        return self.ctx, self.dq, self.dk, self.dv


def inputs(B, L, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v, go = (torch.randn(B, L, d, device="cuda", generator=g) for _ in range(4))
    live = torch.randint(1, L + 1, (B,), device="cuda", generator=g)
    live[0] = L
    return q, k, v, live, go


def time_ms(fns, iters):
    """alternating timed calls: mean ms per call of each fn (CUDA events around each call)"""
    tot = [0.0] * len(fns)
    for _ in range(iters):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            tot[i] += a.elapsed_time(b)
    return [t / iters for t in tot]


def part_a(iters):
    d, H, B = 64, 4, 4096
    for L in (50, 128):
        q, k, v, live, go = inputs(B, L, d, L)
        rt, tl = Attn("rt", q, k, v, live, go, H), Attn("tiled", q, k, v, live, go, H)
        for f in (rt, tl, rt, tl):
            f()
        torch.cuda.synchronize()
        same = all(torch.equal(a, b) for a, b in zip(rt.results(), tl.results()))
        assert same, f"tiled and rt results differ at L={L}"
        ms_rt, ms_tl = time_ms([rt, tl], iters)
        emit(part="a", B=B, L=L, d=d, H=H, bits_equal=same, rt_ms=round(ms_rt, 3), tiled_ms=round(ms_tl, 3),
             tiled_over_rt=round(ms_tl / ms_rt, 3))


def part_b(iters):
    d, rows = 64, 262144
    for L in (200, 512, 1024):
        for dk in (16, 64):
            H, B = d // dk, rows // L
            q, k, v, _, go = inputs(B, L, d, L + dk)
            live = torch.full((B,), L, dtype=torch.int64, device="cuda")
            tl = Attn("tiled", q, k, v, live, go, H)
            tl()
            torch.cuda.synchronize()
            (ms,) = time_ms([tl], iters)
            flop = 14.0 * B * H * (L * (L + 1) / 2) * dk
            emit(part="b", B=B, L=L, d=d, H=H, dk=dk, tiled_fwd_bwd_ms=round(ms, 3), gflop=round(flop / 1e9, 1),
                 tflops=round(flop / ms / 1e9, 2), share_of_fp32_datasheet=round(flop / ms / 1e9 / (FP32_PEAK / 1e12), 3))


# ---------------------------------------------------------------------------------------------------------------------
# (c): whole training steps
# ---------------------------------------------------------------------------------------------------------------------

class StockBlock(nn.Module):
    def __init__(self, d, H):
        super().__init__()
        self.H = H
        self.q, self.k, self.v = nn.Linear(d, d), nn.Linear(d, d), nn.Linear(d, d)
        self.ln1, self.ln2 = nn.LayerNorm(d), nn.LayerNorm(d)
        self.l1, self.l2 = nn.Linear(d, d), nn.Linear(d, d)

    def forward(self, x, keep):
        B, L, d = x.shape
        dk = d // self.H
        split = lambda t: t.view(B, L, self.H, dk).transpose(1, 2)          # noqa: E731
        s = split(self.q(x)) @ split(self.k(x)).transpose(-1, -2) / math.sqrt(dk)
        s = s.masked_fill(~keep, float("-inf"))
        a = torch.softmax(s - s.max(), dim=-1)                             # utils/layers.py's global-max shift
        a = torch.where(torch.isnan(a), torch.zeros_like(a), a)
        c = self.ln1((a @ split(self.v(x))).transpose(1, 2).reshape(B, L, d) + x)
        return self.ln2(self.l2(torch.relu(self.l1(c))) + c)


class StockSASRec(nn.Module):
    def __init__(self, n_items, d, H, layers, hm):
        super().__init__()
        self.i_emb, self.p_emb = nn.Embedding(n_items, d), nn.Embedding(hm + 1, d)
        self.blocks = nn.ModuleList(StockBlock(d, H) for _ in range(layers))

    def load_from(self, kernel_model):
        sd = {k: v.detach().clone() for k, v in kernel_model.state_dict().items()}
        with torch.no_grad():
            self.i_emb.weight.copy_(sd["i_embeddings.weight"])
            self.p_emb.weight.copy_(sd["p_embeddings.weight"])
            for b, blk in enumerate(self.blocks):
                pre = f"transformer_block.{b}."
                for ours, theirs in (("q", "masked_attn_head.q_linear"), ("k", "masked_attn_head.k_linear"),
                                     ("v", "masked_attn_head.v_linear"), ("l1", "linear1"), ("l2", "linear2"),
                                     ("ln1", "layer_norm1"), ("ln2", "layer_norm2")):
                    getattr(blk, ours).weight.copy_(sd[pre + theirs + ".weight"])
                    getattr(blk, ours).bias.copy_(sd[pre + theirs + ".bias"])

    def loss(self, hist, lengths, items):
        B, L = hist.shape
        valid = (hist > 0).long()
        pos = (lengths.view(B, 1) - torch.arange(L, device=hist.device).view(1, L)) * valid
        x = self.i_emb(hist) + self.p_emb(pos)
        keep = torch.ones(L, L, dtype=torch.bool, device=hist.device).tril()
        for blk in self.blocks:
            x = blk(x, keep)
        h = (x * valid.unsqueeze(-1))[torch.arange(B, device=hist.device), lengths - 1]
        pred = (h.unsqueeze(1) * self.i_emb(items)).sum(-1)
        posp, neg = pred[:, :1], pred[:, 1:]
        w = torch.softmax(neg - neg.max(), dim=1)
        return -torch.log(((posp - neg).sigmoid() * w).sum(1).clamp(1e-8, 1 - 1e-8)).mean()


def part_c(iters):
    from rechorus_b200 import plugin
    from rechorus_b200.graph import GraphedStep
    from rechorus_b200.optim import RowSparseOptimizer
    from rechorus_b200.runner import BaseRunner
    n_items, B, K, d, H = 100_000, 4096, 99, 64, 4
    for hm, layers in ((200, 2), (512, 1)):
        p = plugin.SASRec.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
        a = p.parse_args(["--emb_size", str(d), "--num_heads", str(H), "--num_layers", str(layers), "--history_max",
                          str(hm), "--num_neg", str(K), "--tiled_attention", "1", "--table_mode", "fused"])
        a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_long_history.pt"
        torch.manual_seed(0)
        m = plugin.SASRec(a, types.SimpleNamespace(n_users=10, n_items=n_items)).to(a.device)
        stock = StockSASRec(n_items, d, H, layers, hm).cuda()
        stock.load_from(m)
        m.optimizer = RowSparseOptimizer(m, "Adam", lr=1e-3, device_clock=True)
        m.train()
        g = torch.Generator(device="cuda").manual_seed(hm)
        feeds = []
        for _ in range(3):
            lengths = torch.randint(1, hm + 1, (B,), device="cuda", generator=g)
            lengths[0] = hm
            hist = torch.randint(1, n_items, (B, hm), device="cuda", generator=g)
            hist = hist * (torch.arange(hm, device="cuda").view(1, hm) < lengths.view(B, 1))
            feeds.append({"history_items": hist, "lengths": lengths, "batch_size": B, "phase": "train",
                          "item_id": torch.randint(1, n_items, (B, K + 1), device="cuda", generator=g),
                          "user_id": torch.zeros(B, dtype=torch.int64, device="cuda")})
        # first losses on the same weights, before any update
        with torch.no_grad():
            loss0_kernels = float(m.loss(m(feeds[1])))
        opt = torch.optim.Adam(stock.parameters(), lr=1e-3)

        def stock_step(f):
            opt.zero_grad(set_to_none=True)
            ls = stock.loss(f["history_items"], f["lengths"], f["item_id"])
            ls.backward()
            opt.step()
            return ls

        step = GraphedStep(m, feeds[0], warmup=2)                 # two eager steps on feeds[0], then the capture
        l1_k, l2_k = float(step(feeds[1])), float(step(feeds[2]))
        (ms_k,) = time_ms([lambda: step(feeds[2])], iters)
        res = dict(part="c", history_max=hm, blocks=layers, B=B, K=K, d=d, H=H, graphed_step_ms=round(ms_k, 3),
                   kernels_loss_same_weights=round(loss0_kernels, 6),
                   kernels_loss_after_2_and_3_updates=[round(l1_k, 6), round(l2_k, 6)],
                   kernels_peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2**30, 1))
        try:                                                       # the stock step materialises [B, H, L, L] scores
            torch.cuda.reset_peak_memory_stats()
            with torch.no_grad():
                res["stock_loss_same_weights"] = round(float(stock.loss(feeds[1]["history_items"], feeds[1]["lengths"],
                                                                        feeds[1]["item_id"])), 6)
            stock_step(feeds[0])
            stock_step(feeds[0])
            res["stock_loss_after_2_and_3_updates"] = [round(float(stock_step(f).detach()), 6) for f in feeds[1:]]
            (ms_s,) = time_ms([lambda: stock_step(feeds[2])], iters)
            res.update(stock_pytorch_step_ms=round(ms_s, 3), speedup=round(ms_s / ms_k, 2),
                       stock_peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2**30, 1))
        except torch.cuda.OutOfMemoryError:
            res["stock_pytorch_step"] = "out of memory"
        emit(**res)
        if "stock_loss_same_weights" in res:
            # same weights, then the same batches through row-sparse vs dense Adam: the losses agree to 6 digits
            kern = [res["kernels_loss_same_weights"]] + res["kernels_loss_after_2_and_3_updates"]
            stock = [res["stock_loss_same_weights"]] + res["stock_loss_after_2_and_3_updates"]
            assert all(abs(a - b) <= 1e-5 for a, b in zip(kern, stock)), (kern, stock)
        del m, stock, opt, step
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--parts", default="abc")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_history_time.py measures on a CUDA device; none is visible")
    from rechorus_b200 import build
    build.build()
    emit(**card())
    for part, fn in (("a", part_a), ("b", part_b), ("c", part_c)):
        if part in args.parts:
            fn(args.iters)
    emit(**card())


if __name__ == "__main__":
    main()
