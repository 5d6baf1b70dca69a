"""NumPy restatement of the impression setting's evaluation, for tests only: the non-test_all branch of
ImpressionRunner.evaluate + evaluate_method (helpers/ImpressionRunner.py:135-171, :74-133) on a prediction matrix, and the
batches ImpressionModel.Dataset / ImpressionSeqModel.Dataset collate (models/BaseImpressionModel.py:152-184, :200-240).
tests/golden/impression_eval.npz holds what the reference's own code returns on the same inputs."""
import numpy as np


def impression_evaluate(pred, pos_num, neg_num, mp: int, topks, allow_wide_neg: bool = False) -> dict:
    """{NDCG@k for every k, MAP@k for every k, HR@k for every k} -> float64 means over the rows of pred [N, mp + mn]
    (float32; column c < mp is positive slot c, column mp + j negative slot j).  Same array operations in the same
    order as the reference, so the values are equal bit for bit.  mn > mp raises IndexError as the reference does,
    unless allow_wide_neg asks for the same definition extended to those lists (what b2r_impression_metrics computes)."""
    pred = np.asarray(pred, dtype=np.float32)
    N, C = pred.shape
    mn = C - mp
    if mn > mp and not allow_wide_neg:
        raise IndexError("the reference's label matrix is 2 * mp columns wide; mn > mp indexes past it")
    P = np.minimum(np.asarray(pos_num, dtype=np.int64), mp)
    Q = np.minimum(np.asarray(neg_num, dtype=np.int64), mn)
    col = np.arange(C)
    valid = (col < P[:, None]) | ((col >= mp) & (col < mp + Q[:, None]))
    masked = np.where(valid, pred, np.float32(-np.inf))                     # float32, invalid slots -inf
    key = masked - 1e-6 * (col < mp).astype(np.float64)                      # float64: the positive-slot tie breaker
    order = np.argsort(-key, axis=1, kind="mergesort")                      # stable; NaN last
    W = P + Q
    lab = (order < P[:, None]).astype(int)                                   # sorted labels
    lab = lab * (col < W[:, None])                                           # positions past whole_len do not count
    Pm = lab.sum(axis=1)
    ideal = (col < Pm[:, None]).astype(int)                                  # the labels sorted descending

    def dcg(x, k):
        x = x[:, :k]
        return np.sum(x / np.log2(np.arange(2, x.shape[1] + 2)), axis=1)

    def pos_count(k):
        n = Pm.copy()
        n[n == 0] = 1
        n[n > k] = k
        return n

    out = {}
    for k in topks:
        idcg = dcg(ideal, k)
        idcg[idcg == 0] = 1
        out[f"NDCG@{k}"] = (dcg(lab, k) / idcg).mean()
    for k in topks:
        cum = np.cumsum(lab, axis=1)
        cum[:, k:] = 0
        prec = cum / np.arange(1, C + 1)
        out[f"MAP@{k}"] = (np.sum(prec * lab, axis=1) / pos_count(k)).mean()
    for k in topks:
        hits = np.sum(lab[:, :k], axis=1)
        out[f"HR@{k}"] = (hits / pos_count(k) > 0).astype(np.float64).mean()
    return out


def impression_collate(pos_items, neg_items, users, mp: int, mn: int):
    """(user_id int64 [B], item_id int64 [B, mp + mn]) of one batch: [pos[:mp] | 0-pad | neg[:mn] | 0-pad]"""
    B = len(users)
    item_id = np.zeros((B, mp + mn), dtype=np.int64)
    for t in range(B):
        p, n = list(pos_items[t])[:mp], list(neg_items[t])[:mn]
        item_id[t, :len(p)] = p
        item_id[t, mp:mp + len(n)] = n
    return np.asarray(users, dtype=np.int64), item_id


def impression_history(user_his_pos, users, positions, history_max: int):
    """(history_items int64 [B, Lb], lengths int64 [B]) of one ImpressionSeqModel batch: user_his[u]['pos'][:position]
    items, the last history_max of them, right-padded with 0 to the batch's longest"""
    seqs = []
    for u, p in zip(users, positions):
        s = [x[0] for x in user_his_pos[u][:p]]
        if history_max > 0:
            s = s[-history_max:]
        seqs.append(s)
    L = max(len(s) for s in seqs)
    out = np.zeros((len(seqs), L), dtype=np.int64)
    for t, s in enumerate(seqs):
        out[t, :len(s)] = s
    return out, np.array([len(s) for s in seqs], dtype=np.int64)
