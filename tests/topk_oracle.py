"""NumPy restatement of the top-k ordering contract (include/b200rec.h) shared by the CPU and GPU top-k tests.

The reference's save_rec_results (main.py:117-132) keeps sorted(zip(item_id, pred), key=score, reverse=True)[:k] of
every row.  Python's sort is stable, so that is: score descending, ties by candidate column ascending, -0.0 equal to
+0.0.  A stable ascending argsort of -pred gives exactly that order, with -inf (masked entries) after every finite
score in column order and NaN last (NumPy sorts NaN to the end)."""
import numpy as np


def topk_order(pred: np.ndarray, k: int) -> np.ndarray:
    """columns int64 [N, min(k, C)] of each row's top-k list"""
    pred = np.asarray(pred, dtype=np.float32)
    order = np.argsort(-pred, axis=1, kind="stable")
    return order[:, :min(int(k), pred.shape[1])].astype(np.int64)


def topk_rows(pred: np.ndarray, k: int):
    """(columns, scores) as b2r_topk_rows returns them: the scores are pred's own values"""
    cols = topk_order(pred, k)
    return cols, np.take_along_axis(np.asarray(pred, dtype=np.float32), cols, axis=1)


def order_keys(pred: np.ndarray) -> np.ndarray:
    """the 64-bit keys of include/b200rec.h: (~mono(score) << 32) | column, -0.0 folded onto +0.0, NaN last"""
    u = np.asarray(pred, dtype=np.float32).view(np.uint32).copy()
    u[u == 0x80000000] = 0
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    mono = np.where(u & 0x80000000, ~u, u | np.uint32(0x80000000)).astype(np.uint32)
    hi = np.where(nan, np.uint32(0xFFFFFFFF), ~mono).astype(np.uint64)
    cols = np.arange(u.shape[-1], dtype=np.uint64)
    return (hi << np.uint64(32)) | cols


def test_all_matrix(scores_all: np.ndarray, target: np.ndarray, clicked: list) -> np.ndarray:
    """the reference's masked test_all prediction matrix (BaseModel.py:194-198, BaseRunner.py:244-251) from the scores
    of every item [B, n_items]: column 0 is the target's score, column j >= 1 item j's, clicked items -inf"""
    B, n_items = scores_all.shape
    m = scores_all.astype(np.float32).copy()
    m[:, 0] = scores_all[np.arange(B), target]
    for b in range(B):
        c = [j for j in clicked[b] if 1 <= j < n_items]
        m[b, c] = -np.inf
    return m


def planted_rows(rng, N: int, C: int) -> np.ndarray:
    """random rows with planted equal scores, +-0, -inf and NaN"""
    x = rng.standard_normal((N, C)).astype(np.float32)
    x = np.round(x * 4) / 4                                   # many exact ties
    n = max(1, C // 10)
    for r in range(N):
        for val in (0.0, -0.0, -np.inf, np.nan, 1.25):
            x[r, rng.randint(0, C, n)] = val
    return x.astype(np.float32)
