"""CPU: the clicked-set CSR behind the top-k lists, the NumPy restatement of the ordering contract against Python's
own sort, and the argument checks of the new entry points (no GPU needed)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import topk_oracle as T  # noqa: E402


def test_clicked_csr_is_the_sorted_union_with_empty_users():
    from rechorus_b200 import ops
    train = {0: {5, 3}, 1: set(), 2: {9, 1, 4}, 7: {2}}               # user 7 is outside [0, 4): ignored
    residual = {0: {3, 8}, 3: {6}}
    ptr, items = ops.clicked_csr([train, residual], 4)
    assert ptr.tolist() == [0, 3, 3, 6, 7]
    assert items.tolist() == [3, 5, 8, 1, 4, 9, 6]
    ptr, items = ops.clicked_csr([{}, {}], 3)
    assert ptr.tolist() == [0, 0, 0, 0] and len(items) == 1         # one slot so the device buffer is never empty


def test_clicked_sets_holds_the_csr():
    import torch
    from rechorus_b200 import ops
    cs = ops.ClickedSets({1: {4, 2}}, {1: {2, 7}, 0: {1}}, 2, torch.device("cpu"))
    assert cs.n_users == 2 and cs.ptr.tolist() == [0, 1, 4] and cs.items.tolist() == [1, 2, 4, 7]


def test_negative_sampler_csr_unchanged():
    """DeviceNegativeSampler, now built on clicked_csr, holds the CSR its own per-user sort used to build: users in
    [0, n_users) with their training clicks sorted, out-of-range users ignored, at least one item slot"""
    import torch
    from rechorus_b200 import ops
    rng = np.random.RandomState(4)
    n_users, n_items = 30, 200
    clicked = {u: set(rng.randint(1, n_items, rng.randint(0, 15)).tolist()) for u in range(n_users)}
    clicked[n_users + 2] = {7, 9}                                     # outside [0, n_users)
    ptr = np.zeros(n_users + 1, dtype=np.int64)                       # the sampler's former construction
    for u, items in clicked.items():
        if 0 <= int(u) < n_users:
            ptr[int(u) + 1] = len(items)
    ptr = np.cumsum(ptr)
    flat = np.zeros(max(int(ptr[-1]), 1), dtype=np.int64)
    for u, items in clicked.items():
        if 0 <= int(u) < n_users and len(items):
            flat[ptr[int(u)]:ptr[int(u) + 1]] = np.sort(np.fromiter(items, dtype=np.int64, count=len(items)))
    s = ops.DeviceNegativeSampler(clicked, n_users, n_items, torch.device("cpu"), seed=3)
    assert s.ptr.tolist() == ptr.tolist() and s.items.tolist() == flat.tolist()
    assert (s.n_users, s.n_items, s.seed) == (n_users, n_items, 3)
    empty = ops.DeviceNegativeSampler({u: set() for u in range(4)}, 4, n_items, torch.device("cpu"))
    assert empty.ptr.tolist() == [0] * 5 and empty.items.numel() == 1


@pytest.mark.parametrize("C", [1, 2, 7, 100, 1000])
@pytest.mark.parametrize("k", [1, 10, 100])
def test_restatement_equals_python_sorted(C, k):
    """main.py:123-126 row by row (finite scores, ties, +-0, -inf; Python's result is undefined with NaN)"""
    rng = np.random.RandomState(C * 31 + k)
    x = T.planted_rows(rng, 3, C)
    x[np.isnan(x)] = -np.inf
    cols, scores = T.topk_rows(x, k)
    for r in range(x.shape[0]):
        ref = sorted(zip(range(C), x[r]), key=lambda t: t[1], reverse=True)[:k]
        assert cols[r].tolist() == [c for c, _ in ref]
        assert np.array_equal(scores[r].view(np.uint32), np.array([s for _, s in ref], np.float32).view(np.uint32))


@pytest.mark.parametrize("C", [1, 5, 300])
def test_key_order_equals_restatement_with_nan(C):
    """ascending 64-bit key order == the stable argsort of -x, NaN and -inf included"""
    x = T.planted_rows(np.random.RandomState(C), 4, C)
    keys = T.order_keys(x)
    assert np.array_equal(np.argsort(keys, axis=1), T.topk_order(x, C))
    assert (keys[:, :] < np.uint64(0xFFFFFFFFFFFFFFFF)).all()


def test_signed_zero_and_nan_placement():
    x = np.array([[-0.0, 0.0, np.nan, -np.inf, -1.0, np.nan, -np.inf]], np.float32)
    assert T.topk_order(x, 7).tolist() == [[0, 1, 4, 3, 6, 2, 5]]


@pytest.fixture(scope="module")
def handle():
    from rechorus_b200 import build
    from rechorus_b200 import lib as L
    build.build()
    return L.load()


def test_topk_entry_points_reject_null_arguments(handle):
    h = handle
    assert h.b2r_topk_rows(None, 4, 4, 4, 2, None, None, None, 0, None) == -1 and b"null pointer" in h.b2r_last_error()
    assert h.b2r_mask_clicked(None, 4, 4, 4, None, None, None, 3, None, None) == -1
    assert h.b2r_topk_all_items(None, 64, None, 100, 64, None, None, 4, None, None, 3, 10, None, None, None, None, 0,
                                None) == -1


def test_topk_entry_points_reject_k_out_of_range(handle):
    h, p = handle, 256                                       # non-null stand-ins: rejected before any launch
    assert h.b2r_topk_rows(p, 4, 4, 4, 1025, p, p, p, 1 << 20, None) == -3 and b"k=1025" in h.b2r_last_error()
    assert h.b2r_topk_rows(p, 4, 4, 4, 0, p, p, p, 1 << 20, None) == -1
    assert h.b2r_topk_all_items(p, 64, p, 100, 64, p, p, 4, p, p, 3, 1025, p, p, None, p, 1 << 30, None) == -3
    assert h.b2r_topk_all_items(p, 64, p, 100, 64, p, p, 4, p, p, 3, 0, p, p, None, p, 1 << 30, None) == -1
    assert h.b2r_topk_rows_workspace_bytes(4, 100, 1025) == 0 and h.b2r_topk_all_items_workspace_bytes(4, 100, 0) == 0


def test_topk_workspace_sizes(handle):
    h = handle
    assert h.b2r_topk_rows_workspace_bytes(65536, 100, 100) == 0             # one CTA per row, no merge pass
    assert h.b2r_topk_rows_workspace_bytes(2, 1000003, 1024) > 0
    small = h.b2r_topk_all_items_workspace_bytes(4096, 1_000_000, 100)
    assert small == h.b2r_topk_all_items_workspace_bytes(4096, 50_000_000, 100)   # independent of n_items
    assert small < 64 << 20
    assert h.b2r_topk_rows(256, 2, 1000003, 1000003, 100, 256, 256, None, 0, None) == -2


def test_ops_reject_k_before_launch():
    import torch
    from rechorus_b200 import ops
    with pytest.raises(ValueError):
        ops._topk_k(1025)
    with pytest.raises(ValueError):
        ops._topk_k(0)
    from rechorus_b200.lib import B200RecError
    with pytest.raises(B200RecError):
        ops.topk_rows(torch.zeros(2, 3), 1)
