"""CPU: the host side of device-collated SASRec batches -- the history CSR of corpus.user_his (ops.history_csr), the
fixed padded width (ops.history_width), the setup check of DeviceHistory, and the C entry point's argument check."""
import os
import sys
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


def _train_set(corpus, H):
    """plugin.SequentialModel.Dataset over the training rows, with placeholder negatives (they do not enter the history)"""
    from rechorus_b200 import plugin
    model = types.SimpleNamespace(history_max=H, test_all=0, buffer=1)
    ds = plugin.SequentialModel.Dataset(model, corpus, "train")
    ds.data["neg_items"] = np.zeros((len(ds), 1), dtype=np.int64)
    return ds


@pytest.mark.parametrize("H", [8, 3, 0, -1, 10_000])
def test_csr_slices_equal_the_host_feed_dicts(H):
    import fit_corpus
    from rechorus_b200 import ops
    corpus = fit_corpus.build()
    ptr, items = ops.history_csr(corpus.user_his, corpus.n_users)
    assert ptr.dtype == np.int64 and items.dtype == np.int64 and ptr.shape == (corpus.n_users + 1,)
    assert ptr[0] == 0 and ptr[-1] == items.size == sum(len(h) for h in corpus.user_his.values())
    ds = _train_set(corpus, H)
    assert len(ds) > 300
    for i in range(len(ds)):
        u, p = int(ds.data["user_id"][i]), int(ds.data["position"][i])
        n = min(p, H) if H > 0 else p
        want = ds._get_feed_dict(i)["history_items"]
        assert np.array_equal(items[ptr[u] + p - n:ptr[u] + p], want), i
    positions = np.asarray(ds.data["position"], dtype=np.int64)
    top = int(positions.max())
    assert 8 < top < 10_000
    assert ops.history_width(positions, H) == (min(H, top) if H > 0 else top)


def test_width_for_each_history_max():
    from rechorus_b200 import ops
    pos = np.array([3, 1, 7, 2])
    assert ops.history_width(pos, 5) == 5
    assert ops.history_width(pos, 0) == 7 and ops.history_width(pos, -1) == 7
    assert ops.history_width(pos, 50) == 7


def test_csr_keeps_users_without_history_empty():
    from rechorus_b200 import ops
    ptr, items = ops.history_csr({1: [(5, 0), (6, 1)], 3: [(7, 2)]}, 5)
    assert ptr.tolist() == [0, 0, 2, 2, 3, 3] and items.tolist() == [5, 6, 7]
    with pytest.raises(ValueError):
        ops.history_csr({5: [(1, 0)]}, 5)


@pytest.mark.parametrize("bad", ["beyond", "zero"])
def test_a_position_outside_the_history_is_rejected_at_setup(bad):
    import fit_corpus
    import torch
    from rechorus_b200 import ops
    corpus = fit_corpus.build()
    ds = _train_set(corpus, 8)
    users = np.asarray(ds.data["user_id"], dtype=np.int64)
    positions = np.asarray(ds.data["position"], dtype=np.int64).copy()
    positions[5] = len(corpus.user_his[int(users[5])]) + 1 if bad == "beyond" else 0
    with pytest.raises(ValueError, match="position"):
        ops.DeviceHistory(corpus.user_his, corpus.n_users, users, positions, 8, torch.device("cpu"))


def test_collate_history_rejects_a_null_pointer():
    from rechorus_b200 import build
    from rechorus_b200 import lib as L
    build.build()
    h = L.load()
    rc = h.b2r_collate_history(None, None, None, None, 10, None, 0, 4, 8, 8, None, None, None, None)
    assert rc == -1 and b"null pointer" in h.b2r_last_error()
