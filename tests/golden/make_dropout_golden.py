"""Generate tests/golden/{neumf,sasrec}_dropout.npz by executing the UNMODIFIED reference (/root/reference) on CPU, with
each nn.Dropout.forward replaced by x * mask * s, mask = tests.dropout_oracle.dropout_mask of that module's site.

    python tests/golden/make_dropout_golden.py

Shapes are those of neumf_l64_32_16 and sasrec_l2h4 (make_golden.py), p = 0.2.  Each .npz holds the state dict
("w:<key>"), the batch ("in:<key>"), seed / step / p, the per-site masks ("mask:<site>", uint8), the prediction, the loss
and every parameter gradient ("g:<key>").  The SASRec file also holds the same batch right-padded by 7 more columns
("pad:in:history_items") and the reference's outputs for it ("pad:prediction", "pad:loss", "pad:g:<key>").
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import make_golden as MG  # noqa: E402

SEED, STEP, P = 0x9E3779B97F4A7C15, 5, 0.2


def _run(model, batch, site_of, masks_out):
    """forward + loss + backward with every nn.Dropout replaced by x * mask * s (mask keyed by site_of(module, x))"""
    import torch
    from tests import dropout_oracle as D
    s = D.dropout_scale(P)

    def patched(mod, x):
        site, r, t = site_of(mod, x)
        m = D.dropout_mask(SEED, STEP, site, r, t, x.shape[-1], P)
        masks_out[site] = m.reshape(x.shape)
        return x * torch.from_numpy(m.reshape(x.shape)).to(x.dtype) * s

    for mod in model.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.forward = (lambda m: (lambda x: patched(m, x)))(mod)
    model.train()
    model.zero_grad()
    out = model(dict(batch))
    loss = model.loss(out)
    loss.backward()
    grads = {k: (p.grad if p.grad is not None else torch.zeros_like(p)).numpy().copy() for k, p in model.named_parameters()}
    return out["prediction"].detach().numpy().copy(), loss.detach().numpy().copy(), grads


def main():
    import torch
    BPRMF, NeuMF, SASRec, BaseRunner = MG._import_reference()
    g = torch.Generator().manual_seed(20261015)

    def ids(lo, hi, shape):
        return torch.randint(lo, hi, shape, generator=g, dtype=torch.int64)

    def scale_weights(model, scale):
        with torch.no_grad():
            for n, p in model.named_parameters():
                if "layer_norm" not in n:
                    p.mul_(scale)

    # ---------------- NeuMF (NeuMF.py:56-76), neumf_l64_32_16 shape ----------------
    nu, ni, d, layers, B, C, scale = 31, 47, 64, [64, 32, 16], 10, 5, 20.0
    torch.manual_seed(11)
    model = NeuMF(MG._args(NeuMF, BaseRunner, ["--emb_size", str(d), "--layers", str(layers), "--num_neg", str(C - 1),
                                               "--dropout", str(P)]), types_ns(nu, ni))
    scale_weights(model, scale)
    batch = {"user_id": ids(1, nu, (B,)), "item_id": ids(1, ni, (B, C)), "batch_size": B, "phase": "train"}
    calls = [0]

    def neumf_site(mod, x):                       # the one dropout_layer runs after every layer: site = call index
        site = calls[0]
        calls[0] += 1
        return site, np.arange(B * C), np.zeros(B * C)

    masks = {}
    pred, loss, grads = _run(model, batch, neumf_site, masks)
    blob = _blob(model, batch, pred, loss, grads, masks,
                 dict(model="NeuMF", n_users=nu, n_items=ni, d=d, layers=layers, B=B, C=C, scale=scale))
    _save("neumf_dropout", blob)

    # ---------------- SASRec (SASRec.py:51-86, layers.py:112-118), sasrec_l2h4 shape ----------------
    ni, d, L, nl, nh, B, C, scale = 61, 64, 50, 2, 4, 8, 10, 10.0
    torch.manual_seed(13)
    model = SASRec(MG._args(SASRec, BaseRunner, ["--emb_size", str(d), "--history_max", str(L), "--num_layers", str(nl),
                                                 "--num_heads", str(nh), "--num_neg", str(C - 1), "--dropout", str(P)]),
                   types_ns(10, ni))
    scale_weights(model, scale)
    sites = {}
    for i, blk in enumerate(model.transformer_block):
        sites[id(blk.dropout1)], sites[id(blk.dropout2)] = 2 * i, 2 * i + 1
    lengths = ids(1, L - 8, (B,))
    lengths[0] = L - 9                     # ragged; the batch width leaves room for 7 more padding columns
    lengths[1] = 1
    Lb = int(lengths.max())
    hist = ids(1, ni, (B, Lb)) * (torch.arange(Lb).view(1, Lb) < lengths.view(B, 1))
    batch = {"user_id": ids(1, 10, (B,)), "item_id": ids(1, ni, (B, C)), "history_items": hist,
             "history_times": torch.zeros_like(hist), "lengths": lengths, "batch_size": B, "phase": "train"}

    def sasrec_site(mod, x):
        Bx, Lx, _ = x.shape
        b, t = np.meshgrid(np.arange(Bx), np.arange(Lx), indexing="ij")
        return sites[id(mod)], b.reshape(-1), t.reshape(-1)

    masks = {}
    pred, loss, grads = _run(model, batch, sasrec_site, masks)
    blob = _blob(model, batch, pred, loss, grads, masks,
                 dict(model="SASRec", n_items=ni, d=d, history_max=L, num_layers=nl, num_heads=nh, B=B, C=C, scale=scale))
    padded = dict(batch)
    padded["history_items"] = torch.cat([hist, torch.zeros(B, 7, dtype=hist.dtype)], dim=1)
    padded["history_times"] = torch.zeros_like(padded["history_items"])
    pred_p, loss_p, grads_p = _run(model, padded, sasrec_site, {})
    blob["pad:in:history_items"] = padded["history_items"].numpy().copy()
    blob["pad:prediction"], blob["pad:loss"] = pred_p, loss_p
    for k, v in grads_p.items():
        blob["pad:g:" + k] = v
    _save("sasrec_dropout", blob)


def types_ns(nu, ni):
    import types
    return types.SimpleNamespace(n_users=nu, n_items=ni)


def _blob(model, batch, pred, loss, grads, masks, meta):
    import torch
    meta.update(seed=SEED, step=STEP, p=P)
    blob = {"meta": np.array(repr(meta))}
    for k, v in model.state_dict().items():
        blob["w:" + k] = v.detach().numpy().copy()
    for k, v in batch.items():
        if isinstance(v, torch.Tensor):
            blob["in:" + k] = v.numpy().copy()
    for site, m in masks.items():
        blob[f"mask:{site}"] = m.astype(np.uint8)
    blob["prediction"], blob["loss"] = pred, loss
    for k, v in grads.items():
        blob["g:" + k] = v
    return blob


def _save(name, blob):
    path = os.path.join(HERE, name + ".npz")
    np.savez_compressed(path, **blob)
    print(f"{name}: pred {blob['prediction'].shape} loss {float(blob['loss']):.6f} -> {os.path.getsize(path)} B")


if __name__ == "__main__":
    main()
