"""The direct index plan's sort (bucket.cu): a warp per bucket, with the CTA sort for the buckets it defers.  Checked
element for element against the plan's definition (numpy): every bucket's pairs sorted by (row, position) in place,
exactly one row head per touched row -- (row, first position, index of its first pair, run length; 0 for rows with
>= kLong contributions) -- and the long-row list; then two builds of the same ids give the same plan, and the
row-sparse update reads it to the same bits whatever the order of the head list.

Cases: the BASELINE config 2 item and user shapes (counting sort; the user plan alone has few buckets and takes the
one-launch CTA sort), 977 buckets of ~34 pairs (register sort), the config 5 item shape (buckets too wide for a warp:
all deferred), hot rows above kLong and above kRunMax, a skewed batch that spills, n = 1, padding ids.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

K_LONG = 48
K_PAD_D = 32


def _dev():
    return torch.device("cuda", 0)


def _align(x):
    return (x + 255) // 256 * 256


def _layout(n, n_rows):
    """direct_layout (bucket.cu): bucket geometry and the byte offsets of the workspace areas"""
    target = n // 192
    if target < 256:
        target = n // 32
    target = min(max(target, 1), 32768)
    rows_per = (n_rows + target - 1) // target
    shift = 0
    while (1 << shift) < rows_per:
        shift += 1
    nb = (n_rows + (1 << shift) - 1) >> shift
    cap = (3 * (n // nb) + 64 + 63) // 64 * 64
    cap = min(max(cap, 128), 2048)
    L = dict(nb=nb, shift=shift, cap=cap, big_cap=2 * n, spill_cap=n, long_cap=n // K_LONG + 1)
    o = 0
    for name, nbytes in (("cursor", nb * 4 * K_PAD_D), ("counters", 256), ("region", nb * cap * 8),
                         ("big", 2 * n * 8), ("tmp", 2 * n * 8), ("spill", n * 8), ("longs", L["long_cap"] * 8),
                         ("heads", n * 16), ("deferred", nb * 8)):
        L[name] = o
        o += _align(nbytes)
    L["total"] = o
    return L


def _build(ids, n_rows, ignore_id=-1, ignore_n=0):
    """the plan's workspace bytes (host copy) right after b2r_direct_plan_build"""
    from rechorus_b200 import ops
    plan = ops.DirectPlan(ids.to(_dev()), n_rows, ignore_id, ignore_n)
    torch.cuda.synchronize()
    ops.check_ids()
    return plan, plan.ws.cpu().numpy().copy()


def _view(ws, L, name, dtype, count):
    return np.frombuffer(ws[L[name]:L[name] + count * np.dtype(dtype).itemsize].tobytes(), dtype=dtype)


def _decode(ws, L):
    counters = _view(ws, L, "counters", np.int32, 8)
    n_heads, n_long = int(counters[3]), int(counters[2])
    heads = _view(ws, L, "heads", np.uint32, 4 * n_heads).reshape(n_heads, 4).astype(np.int64)
    longs = _view(ws, L, "longs", np.uint32, 2 * n_long).reshape(n_long, 2).astype(np.int64)
    n_pairs = L["nb"] * L["cap"] + L["big_cap"]
    pairs = _view(ws, L, "region", np.uint64, n_pairs)        # regions, then the big area: one index space
    return counters, heads, longs, pairs


def _check(ids, n_rows, ignore_id=-1, ignore_n=0):
    ids = ids.reshape(-1)
    n = ids.numel()
    L = _layout(n, n_rows)
    plan, ws = _build(ids, n_rows, ignore_id, ignore_n)
    assert ws.size == L["total"]
    counters, heads, longs, pairs = _decode(ws, L)
    idn = ids.numpy()
    pos = np.arange(n, dtype=np.int64)
    keep = ~((pos < ignore_n) & (idn == ignore_id))
    want = np.sort((idn[keep].astype(np.uint64) << np.uint64(32)) | pos[keep].astype(np.uint64))
    rows = (want >> np.uint64(32)).astype(np.int64)
    urow, first, runs = np.unique(rows, return_index=True, return_counts=True)

    # one head per touched row: (row, first position, index of the first pair, length or 0 for long rows)
    assert heads.shape[0] == urow.size
    order = np.argsort(heads[:, 0])
    h = heads[order]
    assert np.array_equal(h[:, 0], urow)
    assert np.array_equal(h[:, 1], (want[first] & np.uint64(0xffffffff)).astype(np.int64))
    assert np.array_equal(h[:, 3], np.where(runs >= K_LONG, 0, runs))
    # every row's run sits at its head's index, sorted by position
    idx = np.repeat(h[:, 2], runs) + (np.arange(want.size) - np.repeat(first, runs))
    assert np.array_equal(pairs[idx], want)
    # buckets that kept to their region: the region itself is the sorted bucket
    bucket = rows >> L["shift"]
    bcount = np.bincount(bucket, minlength=L["nb"])
    in_region = bcount[bucket] <= L["cap"]
    ridx = bucket * L["cap"] + (np.arange(want.size) - np.searchsorted(bucket, bucket))
    assert np.array_equal(pairs[ridx[in_region]], want[in_region])
    # long rows: (index of the first pair, length) of every row with >= kLong contributions
    lw = sorted(zip(h[runs >= K_LONG, 2].tolist(), runs[runs >= K_LONG].tolist()))
    assert sorted(map(tuple, longs.tolist())) == lw
    cur = _view(ws, L, "cursor", np.int32, L["nb"] * K_PAD_D)
    assert not cur.any()                                        # cursors left zero for the next plan
    return plan, ws, L, bool((bcount > L["cap"]).any())


def _same_plan(ws1, ws2, L):
    """two builds: same pair array, same head set, same long rows (head / long order may differ)"""
    c1, h1, l1, p1 = _decode(ws1, L)
    c2, h2, l2, p2 = _decode(ws2, L)
    assert np.array_equal(c1[2:4], c2[2:4])
    assert np.array_equal(h1[np.lexsort(h1.T[::-1])], h2[np.lexsort(h2.T[::-1])])
    assert sorted(map(tuple, l1.tolist())) == sorted(map(tuple, l2.tolist()))
    nr = L["nb"] * L["cap"]
    assert np.array_equal(p1[:nr], p2[:nr])


def _apply_bits(plan, ws, L, d=64, seed=3):
    """k_apply_sorted (dense +=) from this plan and from the same plan with its head list reversed: same bits"""
    from rechorus_b200 import ops
    n = plan.n
    g = torch.Generator(device="cpu").manual_seed(seed)
    src = torch.randn(n, d, generator=g).to(_dev())
    coef = torch.randn(n, generator=g).to(_dev())
    srcs = [ops.Source(src=src, n=n, coef=coef)]
    outs = []
    for flip in (False, True):
        w = ws.copy()
        if flip:
            nh = int(_view(w, L, "counters", np.int32, 4)[3])
            a = L["heads"]
            hv = np.frombuffer(w[a:a + 16 * nh].tobytes(), dtype=np.uint32).reshape(nh, 4)[::-1].copy()
            w[a:a + 16 * nh] = np.frombuffer(hv.tobytes(), dtype=np.uint8)
        plan.ws.copy_(torch.from_numpy(w))
        dense = torch.zeros(plan.n_rows, d, device=_dev())
        plan.add_to_dense(dense, srcs)
        outs.append(dense)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    return outs[0]


def _uniform(n, n_rows, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(1, n_rows, (n,), generator=g)


@pytest.mark.parametrize("shape", ["c2_items", "c2_users", "small_buckets", "c5_items"])
def test_plan_matches_definition_at_benchmark_shapes(shape):
    n, n_rows = {"c2_items": (4096 * 100, 1_000_000), "c2_users": (4096, 1_000_000),
                 "small_buckets": (4096 * 8, 1_000_000), "c5_items": (4096 * 256, 25_000_000)}[shape]
    ids = _uniform(n, n_rows, seed={"c2_items": 1, "c2_users": 2, "small_buckets": 4, "c5_items": 3}[shape])
    plan, ws, L, spilled = _check(ids, n_rows)
    assert not spilled
    _, ws2 = _build(ids, n_rows)
    _same_plan(ws, ws2, L)
    if shape != "c5_items":
        _apply_bits(plan, ws, L)


def test_hot_rows_above_kLong_and_kRunMax():
    n, n_rows = 4096 * 100, 1_000_000
    ids = _uniform(n, n_rows, seed=7)
    ids[:100] = 12_345                    # 100 contributions: a long row (>= kLong), the warp defers its bucket
    ids[100:140] = 700_001                # 40 contributions: above kRunMax, below kLong
    ids[140:160] = 500_000                # 20: within the warp's counting sort
    plan, ws, L, _ = _check(ids, n_rows)
    _, ws2 = _build(ids, n_rows)
    _same_plan(ws, ws2, L)
    _apply_bits(plan, ws, L)


def test_long_row_in_a_register_sorted_bucket():
    # n = 32,768 over 1 M rows: 977 buckets of 1,024 rows; bucket 0 gets 50 copies of one row + 10 others (<= 64
    # pairs, the register sort) and lists that row as long
    n, n_rows = 4096 * 8, 1_000_000
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(1024, n_rows, (n,), generator=g)
    ids[:50] = 7
    ids[50:60] = torch.randint(0, 1024, (10,), generator=g)
    plan, ws, L, _ = _check(ids, n_rows)
    assert L["shift"] == 10 and L["nb"] == 977 and _decode(ws, L)[2].shape[0] == 1
    _apply_bits(plan, ws, L)


def test_skewed_batch_spills():
    n, n_rows = 4096 * 100, 1_000_000
    ids = _uniform(n, n_rows, seed=11)
    g = torch.Generator().manual_seed(12)
    ids[::3] = torch.randint(1000, 1400, (len(range(0, n, 3)),), generator=g)    # ~137k pairs in one 512-row bucket
    ids[1::97] = 900_001                                                            # and one very long row
    plan, ws, L, spilled = _check(ids, n_rows)
    assert spilled
    _apply_bits(plan, ws, L)


def test_single_pair():
    plan, ws, L, _ = _check(torch.tensor([4321]), 1_000_000)
    _apply_bits(plan, ws, L)


def test_padding_ids_are_ignored():
    n, n_rows = 4096 * 100, 1_000_000
    ids = _uniform(n, n_rows, seed=13)
    g = torch.Generator().manual_seed(14)
    pad = torch.rand(n, generator=g) < 0.3
    ids[pad] = 0
    plan, ws, L, _ = _check(ids, n_rows, ignore_id=0, ignore_n=n // 2)   # padding only counts in the first half
    _apply_bits(plan, ws, L)
