"""CPU: the host side of device-built evaluation batches -- the per-batch history widths and buffer views against what
collate_batch produces, and the argument checks of ops.rank_all_items_clicked and its C entry point."""
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))


@pytest.mark.parametrize("H", [8, 3, 0, -1, 10_000])
@pytest.mark.parametrize("B", [1, 7, 32, 1000])
def test_history_widths_and_views_equal_collate_batch(H, B):
    """every batch of B consecutive rows: the width eval_history_widths gives is collate_batch's padded width, and the
    [Bn, width] view of the flat buffer is contiguous, fits it and starts at its first element"""
    import fit_corpus
    from rechorus_b200 import ops, plugin
    from rechorus_b200.runner import eval_history_widths, history_view
    corpus = fit_corpus.build()
    model = types.SimpleNamespace(history_max=H, test_all=0, buffer=0)
    ds = plugin.SequentialModel.Dataset(model, corpus, "train")      # the most rows; positions far above H = 3 and 8
    ds.data["neg_items"] = np.zeros((len(ds), 1), dtype=np.int64)
    pos = np.asarray(ds.data["position"], dtype=np.int64)
    assert pos.max() > 8
    lens = np.minimum(pos, H) if H > 0 else pos
    widths = eval_history_widths(lens, B)
    N = len(ds)
    assert len(widths) == (N + B - 1) // B
    flat = torch.empty(B * ops.history_width(pos, H), dtype=torch.int64)
    for bi, start in enumerate(range(0, N, B)):
        rows = range(start, min(N, start + B))
        batch = ds.collate_batch([ds._get_feed_dict(i) for i in rows])
        assert tuple(batch["history_items"].shape) == (len(rows), widths[bi]), bi
        assert np.array_equal(batch["lengths"].numpy(), lens[start:start + len(rows)])
        v = history_view(flat, len(rows), widths[bi])
        assert v.shape == batch["history_items"].shape and v.is_contiguous() and v.data_ptr() == flat.data_ptr()


def test_history_widths_of_no_rows():
    from rechorus_b200.runner import eval_history_widths
    assert eval_history_widths(np.zeros(0, np.int64), 4) == []
    assert eval_history_widths([3, 1, 7, 2, 2], 2) == [3, 7, 2]


def _case(B=4, n_items=20, d=8, n_users=6):
    from rechorus_b200 import ops
    cs = ops.ClickedSets({1: {2, 3}}, {2: {5}}, n_users, "cpu")
    return (torch.zeros(B, d), torch.zeros(n_items, d), torch.ones(B, dtype=torch.int64),
            torch.ones(B, dtype=torch.int64), cs)


def test_rank_all_items_clicked_rejects_cpu_tensors():
    from rechorus_b200 import ops
    from rechorus_b200.lib import B200RecError
    with pytest.raises(B200RecError):
        ops.rank_all_items_clicked(*_case())


@pytest.mark.parametrize("which", ["target", "users", "q_width"])
def test_rank_all_items_clicked_rejects_mismatched_lengths(which):
    from rechorus_b200 import ops
    q, table, target, users, cs = _case()
    if which == "target":
        target = target[:3]
    elif which == "users":
        users = torch.ones(5, dtype=torch.int64)
    else:
        q = torch.zeros(4, 12)
    with pytest.raises(ValueError):
        ops.rank_all_items_clicked(q, table, target, users, cs)


def test_rank_all_items_clicked_rejects_clicked_sets_of_another_size():
    from rechorus_b200 import ops
    q, table, target, users, cs = _case()
    cs.n_users = 9
    with pytest.raises(ValueError, match="n_users"):
        ops.rank_all_items_clicked(q, table, target, users, cs)


def test_entry_point_rejects_bad_arguments_without_a_gpu():
    from rechorus_b200 import build
    from rechorus_b200 import lib as L
    build.build()
    h = L.load()
    assert h.b2r_rank_all_items_clicked(None, 64, None, 100, 64, None, None, 4, None, None, 10, None, None, None,
                                        None) == -1
    assert b"null pointer" in h.b2r_last_error()
