"""Generate tests/golden/impression_fit.npz from the UNMODIFIED reference's own code.  Build container only:

    python tests/golden/make_impression_fit_golden.py

Runs ImpressionRunner.fit (helpers/ImpressionRunner.py:173-197) for two seeded epochs over ImpressionModel.Dataset and
ImpressionSeqModel.Dataset (models/BaseImpressionModel.py) on a ragged toy corpus, with a stub model that records what fit
passes it: every batch's ``user_id``, ``item_id``, labels and (sequential) ``history_items`` / ``lengths``, in the order
the DataLoader yields them, and the global CPU RNG state after each epoch.  The corpus has N not a multiple of B,
mn > mp, pos_num > mp and lists longer than mp / mn.  The general Dataset runs with num_workers 0, the sequential one
with 2.
"""
import os
import sys
import types

import numpy as np

REF_SRC = os.environ.get("B2R_REFERENCE_SRC", "/root/reference/src")
OUT = os.path.dirname(os.path.abspath(__file__))

MP, MN, B, H, SEED, EPOCHS = 3, 5, 5, 3, 2024, 2
WORKERS = {"general": 0, "seq": 2}


def corpus():
    """(rows, user_his, n_users, n_items): rows are (user, positives, negatives, position, neg_position); a user's
    history lists hold the items of their earlier rows"""
    rng = np.random.RandomState(29)
    n_users, n_items = 8, 50
    rows, user_his = [], {}
    for u in range(1, n_users):
        user_his[u] = {"pos": [], "neg": []}
        for _ in range(rng.randint(2, 6)):
            pos = [int(i) for i in rng.randint(1, n_items, rng.randint(1, MP + 3))]
            neg = [int(i) for i in rng.randint(1, n_items, rng.randint(1, MN + 4))]
            rows.append((u, pos, neg, len(user_his[u]["pos"]), len(user_his[u]["neg"])))
            t = len(rows)
            user_his[u]["pos"] += [(i, t) for i in pos]
            user_his[u]["neg"] += [(i, t) for i in neg]
    return rows, user_his, n_users, n_items


class StubModel:
    """what ImpressionRunner.fit and the two Datasets read of a model; forward and loss record their inputs"""

    def __init__(self):
        self.device = None
        self.test_all, self.buffer = 0, 0
        self.train_max_pos_item = self.test_max_pos_item = MP
        self.train_max_neg_item = self.test_max_neg_item = MN
        self.history_max = H
        self.optimizer = types.SimpleNamespace(zero_grad=lambda: None, step=lambda: None)
        self.batches = []

    def train(self, mode=True):
        return self

    def __call__(self, batch):
        import torch
        self.batches.append({k: v.clone() for k, v in batch.items() if isinstance(v, torch.Tensor)})
        return {"prediction": torch.zeros(batch["item_id"].shape)}

    def loss(self, out_dict, target=None):
        import torch
        self.batches[-1]["labels"] = target.clone()
        return torch.zeros((), requires_grad=True)


def main():
    np.object, np.int, np.float = object, int, float
    sys.path.insert(0, REF_SRC)
    import pandas as pd
    import torch

    from helpers.ImpressionRunner import ImpressionRunner
    from models.BaseImpressionModel import ImpressionModel, ImpressionSeqModel
    rows, user_his, n_users, n_items = corpus()
    df = pd.DataFrame({"user_id": [r[0] for r in rows], "pos_items": [r[1] for r in rows],
                       "neg_items": [r[2] for r in rows], "pos_num": [len(r[1]) for r in rows],
                       "neg_num": [len(r[2]) for r in rows], "position": [r[3] for r in rows],
                       "neg_position": [r[4] for r in rows], "time": list(range(len(rows)))})
    corp = types.SimpleNamespace(data_df={"train": df}, user_his=user_his, n_users=n_users, n_items=n_items)
    blob = {"user_id": df.user_id.to_numpy(np.int64), "position": df.position.to_numpy(np.int64),
            "pos_ptr": np.cumsum([0] + [len(r[1]) for r in rows]).astype(np.int64),
            "pos_flat": np.array([i for r in rows for i in r[1]], dtype=np.int64),
            "neg_ptr": np.cumsum([0] + [len(r[2]) for r in rows]).astype(np.int64),
            "neg_flat": np.array([i for r in rows for i in r[2]], dtype=np.int64),
            "his_users": np.array(sorted(user_his), dtype=np.int64),
            "his_ptr": np.cumsum([0] + [len(user_his[u]["pos"]) for u in sorted(user_his)]).astype(np.int64),
            "his_flat": np.array([x[0] for u in sorted(user_his) for x in user_his[u]["pos"]], dtype=np.int64),
            "n_users": np.int64(n_users), "mp": np.int64(MP), "mn": np.int64(MN), "B": np.int64(B),
            "history_max": np.int64(H), "seed": np.int64(SEED), "epochs": np.int64(EPOCHS)}
    for tag, cls in (("general", ImpressionModel), ("seq", ImpressionSeqModel)):
        model = StubModel()
        ds = cls.Dataset(model, corp, "train")
        N = len(ds)
        assert N % B != 0
        runner = ImpressionRunner.__new__(ImpressionRunner)
        runner.batch_size, runner.num_workers, runner.pin_memory = B, WORKERS[tag], 0
        blob[f"{tag}/rows"], blob[f"{tag}/num_workers"] = np.int64(N), np.int64(WORKERS[tag])
        torch.manual_seed(SEED)
        for e in range(1, EPOCHS + 1):
            model.batches = []
            loss = ImpressionRunner.fit(runner, ds, epoch=e)
            assert loss == 0.0 and len(model.batches) == (N + B - 1) // B
            blob[f"{tag}/{e}/rng"] = torch.get_rng_state().numpy()
            for bi, b in enumerate(model.batches):
                for k in ("user_id", "item_id", "labels") + (("history_items", "lengths") if tag == "seq" else ()):
                    blob[f"{tag}/{e}/{bi}/{k}"] = b[k].numpy()
        print(tag, N, "rows")
    np.savez_compressed(os.path.join(OUT, "impression_fit.npz"), **blob)


if __name__ == "__main__":
    main()
