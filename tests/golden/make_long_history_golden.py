"""Generate tests/golden/sasrec_long.npz by executing the UNMODIFIED reference (/root/reference) on CPU: SASRec at
history_max 200 with 2 blocks, d = 64, H = 4 -- a width only --tiled_attention trains -- with p = 0.2 (each nn.Dropout
replaced by x * mask * s, mask = tests.dropout_oracle.dropout_mask of its site, as make_dropout_golden.py does) and the
same weights and batch at p = 0.

    python tests/golden/make_long_history_golden.py

Keys as in make_dropout_golden.py ("w:", "in:", "prediction", "loss", "g:", meta with seed / step / p); the p = 0 results
are stored under "p0:prediction", "p0:loss" and "p0:g:<key>".  The batch is ragged, its widest history is 200, and one
history is a single item.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

import make_dropout_golden as MD  # noqa: E402
import make_golden as MG  # noqa: E402


def main():
    import torch
    _, _, SASRec, BaseRunner = MG._import_reference()
    g = torch.Generator().manual_seed(20261017)

    def ids(lo, hi, shape):
        return torch.randint(lo, hi, shape, generator=g, dtype=torch.int64)

    ni, d, L, nl, nh, B, C, scale = 97, 64, 200, 2, 4, 6, 8, 3.0

    def model_at(p):
        torch.manual_seed(17)
        m = SASRec(MG._args(SASRec, BaseRunner, ["--emb_size", str(d), "--history_max", str(L), "--num_layers", str(nl),
                                                 "--num_heads", str(nh), "--num_neg", str(C - 1), "--dropout", str(p)]),
                   MD.types_ns(10, ni))
        with torch.no_grad():
            for n, q in m.named_parameters():
                if "layer_norm" not in n:
                    q.mul_(scale)
        return m

    model = model_at(MD.P)
    sites = {}
    for i, blk in enumerate(model.transformer_block):
        sites[id(blk.dropout1)], sites[id(blk.dropout2)] = 2 * i, 2 * i + 1
    lengths = ids(1, L + 1, (B,))
    lengths[0], lengths[1], lengths[2] = L, 1, 129
    hist = ids(1, ni, (B, L)) * (torch.arange(L).view(1, L) < lengths.view(B, 1))
    batch = {"user_id": ids(1, 10, (B,)), "item_id": ids(1, ni, (B, C)), "history_items": hist,
             "history_times": torch.zeros_like(hist), "lengths": lengths, "batch_size": B, "phase": "train"}

    def sasrec_site(mod, x):
        Bx, Lx, _ = x.shape
        b, t = np.meshgrid(np.arange(Bx), np.arange(Lx), indexing="ij")
        return sites[id(mod)], b.reshape(-1), t.reshape(-1)

    pred, loss, grads = MD._run(model, batch, sasrec_site, {})
    blob = MD._blob(model, batch, pred, loss, grads, {},
                    dict(model="SASRec", n_items=ni, d=d, history_max=L, num_layers=nl, num_heads=nh, B=B, C=C,
                         scale=scale))
    model0 = model_at(0.0)
    model0.load_state_dict(model.state_dict())
    model0.train()
    model0.zero_grad()
    out = model0(dict(batch))
    loss0 = model0.loss(out)
    loss0.backward()
    blob["p0:prediction"] = out["prediction"].detach().numpy().copy()
    blob["p0:loss"] = loss0.detach().numpy().copy()
    for k, q in model0.named_parameters():
        blob["p0:g:" + k] = (q.grad if q.grad is not None else torch.zeros_like(q)).numpy().copy()
    MD._save("sasrec_long", blob)


if __name__ == "__main__":
    main()
