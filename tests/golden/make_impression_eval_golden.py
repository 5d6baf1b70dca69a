"""Generate tests/golden/impression_eval.npz from the UNMODIFIED reference's own code.  Build container only:

    python tests/golden/make_impression_eval_golden.py

(a) ImpressionRunner.evaluate (helpers/ImpressionRunner.py:135-171, with evaluate_method :74-133) on seeded float32
    predictions, through a stub dataset and a runner whose predict() returns them: keys "ev/<case>/...", the metric dict
    as parallel arrays of key names (in order) and float64 values.
(b) The batches ImpressionModel.Dataset and ImpressionSeqModel.Dataset collate (models/BaseImpressionModel.py:152-184,
    :200-240) on a tiny synthetic impression corpus with ragged lists longer than mp / mn: keys "col/...".
"""
import os
import sys
import types

import numpy as np

REF_SRC = os.environ.get("B2R_REFERENCE_SRC", "/root/reference/src")
OUT = os.path.dirname(os.path.abspath(__file__))

# name -> (rows, mp, mn, cut-offs, score kind)
EVAL_CASES = {
    "ties": (300, 20, 20, [1, 3, 5, 10, 20], "int"),
    "specials": (240, 8, 5, [1, 3, 5, 50], "special"),
    "one_one": (120, 1, 1, [1, 2, 10], "int"),
    "narrow_neg": (200, 20, 7, [2, 5, 10, 40, 100], "normal"),
    "many_k": (400, 3, 3, [1, 2, 3, 4, 5, 6, 7, 10, 1000], "int"),
}


def eval_inputs(name):
    N, mp, mn, ks, kind = EVAL_CASES[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    C = mp + mn
    if kind == "int":
        pred = rng.randint(0, 4, (N, C)).astype(np.float32)
    elif kind == "normal":
        pred = rng.randn(N, C).astype(np.float32)
    else:
        pred = rng.randint(-2, 3, (N, C)).astype(np.float32) * np.float32(0.5)
        pick = rng.rand(N, C)
        pred[pick < 0.08] = -np.inf
        pred[(pick >= 0.08) & (pick < 0.14)] = np.nan
        pred[(pick >= 0.14) & (pick < 0.18)] = np.inf
        pred[(pick >= 0.18) & (pick < 0.24)] = -0.0
    pos_num = rng.randint(0, mp + 4, N).astype(np.int64)            # beyond mp, and 0
    neg_num = rng.randint(0, mn + 4, N).astype(np.int64)
    return pred, pos_num, neg_num, mp, mn, ks


def run_evaluate(pred, pos_num, neg_num, mp, mn, ks):
    from helpers.ImpressionRunner import ImpressionRunner
    runner = ImpressionRunner.__new__(ImpressionRunner)
    runner.predict = lambda data: pred.copy()
    model = types.SimpleNamespace(test_all=0, test_max_pos_item=mp, test_max_neg_item=mn)
    data = types.SimpleNamespace(model=model, corpus=None, neg_len=mn,
                                 data={"user_id": list(range(len(pred))), "pos_num": list(pos_num),
                                       "neg_num": list(neg_num)})
    return ImpressionRunner.evaluate(runner, data, ks, ["NDCG", "HR"])


# (b): a tiny impression corpus; rows are (user, positives, negatives), histories per user are the earlier positives
COL_MP, COL_MN, COL_B, COL_H = 4, 3, 4, 3


def collate_corpus():
    rng = np.random.RandomState(11)
    n_users, n_items = 7, 40
    rows, user_his = [], {}
    for u in range(1, n_users):
        user_his[u] = {"pos": [], "neg": []}
        for _ in range(rng.randint(2, 5)):
            pos = list(rng.randint(1, n_items, rng.randint(1, COL_MP + 3)))
            neg = list(rng.randint(1, n_items, rng.randint(1, COL_MN + 4)))
            rows.append((u, pos, neg, len(user_his[u]["pos"]), len(user_his[u]["neg"])))
            t = len(rows)
            user_his[u]["pos"] += [(int(i), t) for i in pos]
            user_his[u]["neg"] += [(int(i), t) for i in neg]
    return rows, user_his, n_users, n_items


def run_collate():
    import pandas as pd
    from models.BaseImpressionModel import ImpressionModel, ImpressionSeqModel
    rows, user_his, n_users, n_items = collate_corpus()
    df = pd.DataFrame({"user_id": [r[0] for r in rows], "pos_items": [r[1] for r in rows],
                       "neg_items": [r[2] for r in rows], "pos_num": [len(r[1]) for r in rows],
                       "neg_num": [len(r[2]) for r in rows], "position": [r[3] for r in rows],
                       "neg_position": [r[4] for r in rows], "time": list(range(len(rows)))})
    corpus = types.SimpleNamespace(data_df={"dev": df}, user_his=user_his, n_users=n_users, n_items=n_items)
    model = types.SimpleNamespace(test_all=0, buffer=0, test_max_pos_item=COL_MP, test_max_neg_item=COL_MN,
                                  train_max_pos_item=COL_MP, train_max_neg_item=COL_MN, history_max=COL_H)
    blob = {"col/user_id": df.user_id.to_numpy(np.int64), "col/position": df.position.to_numpy(np.int64),
            "col/pos_ptr": np.cumsum([0] + [len(r[1]) for r in rows]).astype(np.int64),
            "col/pos_flat": np.array([i for r in rows for i in r[1]], dtype=np.int64),
            "col/neg_ptr": np.cumsum([0] + [len(r[2]) for r in rows]).astype(np.int64),
            "col/neg_flat": np.array([i for r in rows for i in r[2]], dtype=np.int64),
            "col/his_users": np.array(sorted(user_his), dtype=np.int64),
            "col/his_ptr": np.cumsum([0] + [len(user_his[u]["pos"]) for u in sorted(user_his)]).astype(np.int64),
            "col/his_flat": np.array([x[0] for u in sorted(user_his) for x in user_his[u]["pos"]], dtype=np.int64),
            "col/n_users": np.int64(n_users), "col/mp": np.int64(COL_MP), "col/mn": np.int64(COL_MN),
            "col/B": np.int64(COL_B), "col/history_max": np.int64(COL_H)}
    for tag, cls in (("general", ImpressionModel), ("seq", ImpressionSeqModel)):
        ds = cls.Dataset(model, corpus, "dev")
        N = len(ds)
        blob[f"col/{tag}/rows"] = np.int64(N)
        for bi, start in enumerate(range(0, N, COL_B)):
            feed = ds.collate_batch([ds[i] for i in range(start, min(N, start + COL_B))])
            blob[f"col/{tag}/{bi}/user_id"] = feed["user_id"].numpy()
            blob[f"col/{tag}/{bi}/item_id"] = feed["item_id"].numpy()
            if tag == "seq":
                blob[f"col/{tag}/{bi}/history_items"] = feed["history_items"].numpy()
                blob[f"col/{tag}/{bi}/lengths"] = feed["lengths"].numpy()
    return blob


def main():
    np.object, np.int, np.float = object, int, float
    sys.path.insert(0, REF_SRC)
    blob = {}
    for name in EVAL_CASES:
        pred, pos_num, neg_num, mp, mn, ks = eval_inputs(name)
        res = run_evaluate(pred, pos_num, neg_num, mp, mn, ks)
        blob[f"ev/{name}/pred"], blob[f"ev/{name}/pos_num"], blob[f"ev/{name}/neg_num"] = pred, pos_num, neg_num
        blob[f"ev/{name}/mp"], blob[f"ev/{name}/topk"] = np.int64(mp), np.array(ks, dtype=np.int64)
        blob[f"ev/{name}/keys"] = np.array(list(res.keys()))
        blob[f"ev/{name}/values"] = np.array([float(v) for v in res.values()], dtype=np.float64)
        print(name, res)
    blob.update(run_collate())
    np.savez_compressed(os.path.join(OUT, "impression_eval.npz"), **blob)


if __name__ == "__main__":
    main()
