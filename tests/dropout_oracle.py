"""CPU restatement of the fused dropout (include/b200rec.h, b2r_dropout; csrc/dropout.cuh) -- test infrastructure, the
checker of the kernels' mask bits -- and of NeuMF / SASRec with given dropout masks (NeuMF.py:69-72, layers.py:112-118),
on top of oracle/rechorus_oracle.py.

Element (row r, position t, column j) of dropout site ``site`` at training step ``step``:
    word = Philox4x32-10(ctr = (r, (t << 16) | (j >> 2), 0x80000000 | site, lo32(step)), key = (lo32(seed), hi32(seed)))[j & 3]
    kept iff word >= floor(p * 2^32); a kept element is scaled by float(1 / (1 - p)) (0 at p = 1).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import rechorus_oracle as O

_M0, _M1, _W0, _W1, _MASK = (np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85),
                             np.uint64(0xFFFFFFFF))


def philox4x32_10_np(c0, c1, c2, c3, k0, k1):
    """O.philox4x32_10 over numpy arrays (every value a 32-bit word held in uint64); returns the four output words"""
    c = [np.asarray(v, dtype=np.uint64) & _MASK for v in (c0, c1, c2, c3)]
    k = [np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)]
    for _ in range(10):
        p0, p1 = _M0 * c[0], _M1 * c[2]                     # 32 x 32 bits: exact in uint64
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & _MASK]
        k = [(k[0] + _W0) & _MASK, (k[1] + _W1) & _MASK]
    return c


def dropout_scale(p: float) -> float:
    return 0.0 if p >= 1.0 else float(np.float32(1.0 / (1.0 - p)))


def dropout_mask(seed: int, step: int, site: int, r, t, ncols: int, p: float) -> np.ndarray:
    """uint8 [n, ncols] keep mask of the activation rows with logical coordinates (r[i], t[i])"""
    r = np.asarray(r, dtype=np.uint64).reshape(-1, 1)
    t = np.asarray(t, dtype=np.uint64).reshape(-1, 1)
    j = np.arange(ncols, dtype=np.uint64).reshape(1, -1)
    n = r.shape[0]
    ones = np.ones((n, ncols), dtype=np.uint64)
    words = philox4x32_10_np(r * ones, (t << np.uint64(16)) | (j >> np.uint64(2)),
                             ones * np.uint64(0x80000000 | site), ones * np.uint64(step & 0xFFFFFFFF),
                             seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    sel = (j & np.uint64(3)).astype(np.int64) * ones.astype(np.int64)
    word = np.choose(sel, words)
    thr = int(np.floor(p * 4294967296.0))
    return (word >= np.uint64(thr) if thr < (1 << 32) else np.zeros_like(word, dtype=bool)).astype(np.uint8)


def neumf_mask(seed, step, layer, B, C, width, p):
    """[B*C, width]: row r = b*C + c, t = 0, site = layer"""
    return dropout_mask(seed, step, layer, np.arange(B * C), np.zeros(B * C), width, p)


def sasrec_mask(seed, step, site, B, L, d, p):
    """[B, L, d]: row (b, t), site 2i (dropout1) / 2i+1 (dropout2) of block i"""
    b, t = np.meshgrid(np.arange(B), np.arange(L), indexing="ij")
    return dropout_mask(seed, step, site, b.reshape(-1), t.reshape(-1), d, p).reshape(B, L, d)


# ------------------------------------------------------------------------------------------------------
# the models with explicit masks (float tensors of 0 / 1), restated from oracle/rechorus_oracle.py
# ------------------------------------------------------------------------------------------------------

def neumf_scores(p, user_id, item_id, masks, s):
    """NeuMF.py:56-76 with self.dropout_layer(x) = x * masks[l] * s after layer l's ReLU (masks[l]: [B*C, w])"""
    B, C = item_id.shape
    uid = user_id.view(B, 1).expand(B, C)
    mf = F.embedding(uid, p["mf_u_embeddings.weight"]) * F.embedding(item_id, p["mf_i_embeddings.weight"])
    h = torch.cat([F.embedding(uid, p["mlp_u_embeddings.weight"]), F.embedding(item_id, p["mlp_i_embeddings.weight"])], dim=-1)
    l = 0
    while f"mlp.{l}.weight" in p:
        h = torch.relu(F.linear(h, p[f"mlp.{l}.weight"], p[f"mlp.{l}.bias"]))
        h = h * masks[l].view(B, C, -1).to(h.dtype) * s
        l += 1
    return F.linear(torch.cat([mf, h], dim=-1), p["prediction.weight"]).reshape(B, C)


def _block(x, p, pre, num_heads, m1, m2, s):
    """O._attention_block with layers.py:113,117's dropout1 / dropout2 as x * mask * s"""
    B, L, d = x.shape
    dk = d // num_heads

    def heads(name):
        y = F.linear(x, p[pre + f"masked_attn_head.{name}.weight"], p[pre + f"masked_attn_head.{name}.bias"])
        return y.view(B, L, num_heads, dk).permute(0, 2, 1, 3)

    q, k, v = heads("q_linear"), heads("k_linear"), heads("v_linear")
    sc = (q @ k.transpose(-1, -2)) / dk ** 0.5
    keep = torch.ones(L, L, dtype=torch.bool).tril()
    sc = sc.masked_fill(~keep, float("-inf"))
    a = torch.softmax(sc - sc.max(), dim=-1)
    a = torch.where(torch.isnan(a), torch.zeros_like(a), a)
    ctx = (a @ v).permute(0, 2, 1, 3).reshape(B, L, d)
    c = F.layer_norm(ctx * m1 * s + x, (d,), p[pre + "layer_norm1.weight"], p[pre + "layer_norm1.bias"], 1e-5)
    o = F.linear(torch.relu(F.linear(c, p[pre + "linear1.weight"], p[pre + "linear1.bias"])),
                 p[pre + "linear2.weight"], p[pre + "linear2.bias"])
    return F.layer_norm(o * m2 * s + c, (d,), p[pre + "layer_norm2.weight"], p[pre + "layer_norm2.bias"], 1e-5)


def sasrec_scores(p, history, lengths, item_id, num_heads, masks, s):
    """SASRec.py:51-81 with masks[site] [B, L, d] for site 2i / 2i+1 of block i"""
    B, L = history.shape
    valid = (history > 0).to(torch.long)
    pos = (lengths.view(B, 1) - torch.arange(L).view(1, L)) * valid
    x = F.embedding(history, p["i_embeddings.weight"]) + F.embedding(pos, p["p_embeddings.weight"])
    b = 0
    while f"transformer_block.{b}.linear1.weight" in p:
        x = _block(x, p, f"transformer_block.{b}.", num_heads, masks[2 * b].to(x.dtype), masks[2 * b + 1].to(x.dtype), s)
        b += 1
    x = x * valid.unsqueeze(-1).to(x.dtype)
    h = x[torch.arange(B), lengths - 1]
    return torch.einsum("bd,bcd->bc", h, F.embedding(item_id, p["i_embeddings.weight"]))


def loss_and_grads(model, p, batch, masks, s, num_heads=4):
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in p.items()}
    if model == "NeuMF":
        pred = neumf_scores(leaves, batch["user_id"], batch["item_id"], masks, s)
    else:
        pred = sasrec_scores(leaves, batch["history_items"], batch["lengths"], batch["item_id"], num_heads, masks, s)
    loss = O.bpr_loss(pred)
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in leaves.items()}
    return pred.detach(), loss.detach(), grads
