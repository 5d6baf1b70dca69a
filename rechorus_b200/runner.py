"""Stand-alone mirror of the reference's runner surface (helpers/BaseRunner.py) for use without the
reference checkout: same flags, same ``train / fit / evaluate / predict / evaluate_method / print_res``
semantics, same CPU RNG stream for the per-batch candidate shuffle.  Additions (all opt-in flags):
``--fused_optimizer 1`` installs ``RowSparseOptimizer`` through the ``model.optimizer`` seam
(BaseRunner.py:176-177) and switches the embedding tables to 'fused' gradient mode.
"""
from __future__ import annotations

import gc
import logging
import os
from concurrent.futures import ThreadPoolExecutor
from time import time
from typing import Dict, List

import numpy as np
import torch
from torch.utils.data import DataLoader

from . import ops
from .optim import RowSparseOptimizer


def batch_to_device(batch: dict, device) -> dict:
    # utils/utils.py:30-34
    for k, v in batch.items():
        if isinstance(v, torch.Tensor):
            batch[k] = v.to(device)
    return batch


def format_metric(result: Dict[str, float]) -> str:
    # utils/utils.py:54-69: "HR@5:0.1234,NDCG@5:0.0567" sorted by k then metric name
    keys = sorted(result, key=lambda s: (int(s.split("@")[1]) if "@" in s else 0, s.split("@")[0]))
    parts = []
    for k in keys:
        v = result[k]
        parts.append(f"{k}:{v:<.4f}" if isinstance(v, (float, np.floating)) else f"{k}:{v}")
    return ",".join(parts)


def _poll_ids(model) -> None:
    """One synchronising poll of the kernels' out-of-range-id counter per epoch / evaluation: the reference's
    nn.Embedding raises IndexError on a bad id (BPRMF.py:39-40); the kernels clamp and count, so the runner raises."""
    dev = getattr(model, "device", None)
    if isinstance(dev, torch.device) and dev.type == "cuda":
        ops.check_ids(dev if dev.index is not None else None)


def eval_history_widths(lengths, B: int) -> List[int]:
    """The history width of each evaluation batch of B consecutive rows: the longest history in it, the width
    collate_batch's pad_sequence (or np.array, when all are equal) gives (BaseModel.py:135-152).  lengths: the rows'
    min(position, history_max) (the whole position when history_max <= 0)."""
    lengths = np.asarray(lengths, dtype=np.int64)
    if lengths.size == 0:
        return []
    return [int(w) for w in np.maximum.reduceat(lengths, np.arange(0, lengths.size, int(B)))]


def history_view(flat: torch.Tensor, Bn: int, width: int) -> torch.Tensor:
    """A contiguous [Bn, width] batch of histories at the start of one preallocated flat buffer"""
    return flat[:Bn * width].view(Bn, width)


def _eval_state(dataset, B: int) -> dict:
    """The device inputs of one evaluation phase, uploaded when a device route first evaluates it and cached on the
    dataset (as fit_on_device caches its state): user / target columns, the fixed neg_items (unless test_all), the
    clicked-item CSR (test_all), the history CSR (sequential models), and batch buffers for eval_batch_size B."""
    model = dataset.model
    st = dataset.__dict__.get("_b2r_eval")
    dev = model.device
    corpus, data = dataset.corpus, dataset.data
    test_all = bool(model.test_all)
    if st is None:
        st = {"users": torch.as_tensor(np.asarray(data["user_id"], dtype=np.int64)).to(dev),
              "targets": torch.as_tensor(np.asarray(data["item_id"], dtype=np.int64)).to(dev), "B": None}
        if test_all:
            st["clicked"] = ops.ClickedSets(corpus.train_clicked_set, corpus.residual_clicked_set, corpus.n_users, dev)
        if hasattr(model, "history_max"):
            st["his"] = ops.DeviceHistory(corpus.user_his, corpus.n_users, data["user_id"], data["position"],
                                          model.history_max, dev)
            pos = np.asarray(data["position"], dtype=np.int64)
            H = int(model.history_max)
            st["lens"] = np.minimum(pos, H) if H > 0 else pos    # BaseModel.py:240-242's slice lengths
        dataset.__dict__["_b2r_eval"] = st
    N = st["users"].numel()
    if not test_all and st.get("neg_src") is not data["neg_items"]:
        st["neg"] = torch.as_tensor(np.asarray(data["neg_items"], dtype=np.int64).reshape(N, -1)).to(dev)
        st["neg_src"] = data["neg_items"]
        st["B"] = None
    if st["B"] != B:
        bufs = {"user_id": torch.empty(B, dtype=torch.int64, device=dev)}
        if not test_all:
            bufs["item_id"] = torch.empty((B, st["neg"].shape[1] + 1), dtype=torch.int64, device=dev)
        elif not model.has_query_rows():                  # [target | arange(1, n_items)], column 0 per batch
            bufs["item_id"] = torch.arange(corpus.n_items, dtype=torch.int64, device=dev).repeat(B, 1)
        if "his" in st:
            # pad_sequence pads to the batch maximum: each batch's [Bn, Lb] is a contiguous view of one buffer
            bufs["history_items"] = torch.empty(B * st["his"].width, dtype=torch.int64, device=dev)
            bufs["lengths"] = torch.empty(B, dtype=torch.int64, device=dev)
            st["widths"] = eval_history_widths(st["lens"], B)
        st["bufs"], st["B"] = bufs, B
    return st


def device_eval_batches(dataset, B: int):
    """Yields (feed dict, clicked sets or None) for the batches of B rows of an evaluation phase (a model's Dataset), in
    dataset order, built on the device with the same values collate_batch gives (BaseModel.py:135-152,192-203,236-245):
    b2r_collate_general for the 1 + K candidates, the targets alone for a dot-product model under test_all, a
    [target | arange(1, n_items)] matrix for other models under test_all, and for sequential models the histories
    right-padded to the batch's longest one (b2r_collate_history).  Consecutive batches share the buffers: a batch
    must be consumed (its work enqueued on the current stream) before the next one is requested."""
    model = dataset.model
    B = int(B)
    st = _eval_state(dataset, B)
    bufs, his, clicked = st["bufs"], st.get("his"), st.get("clicked")
    users, targets = st["users"], st["targets"]
    N, test_all = users.numel(), bool(model.test_all)
    for bi, start in enumerate(range(0, N, B)):
        Bn = min(B, N - start)
        feed = {"batch_size": Bn, "phase": dataset.phase}
        if not test_all:
            ops.collate_general(users, targets, st["neg"], None, start, Bn, bufs["user_id"], bufs["item_id"])
            feed["user_id"], feed["item_id"] = bufs["user_id"][:Bn], bufs["item_id"][:Bn]
        else:
            feed["user_id"] = users[start:start + Bn]
            tgt = targets[start:start + Bn].view(-1, 1)
            if "item_id" in bufs:
                bufs["item_id"][:Bn, :1].copy_(tgt)
                feed["item_id"] = bufs["item_id"][:Bn]
            else:
                feed["item_id"] = tgt
        if his is not None:
            hb = history_view(bufs["history_items"], Bn, st["widths"][bi])
            his.collate(users, None, start, Bn, hb, bufs["lengths"])
            feed["history_items"], feed["lengths"] = hb, bufs["lengths"][:Bn]
        yield feed, clicked


def _impression_state(dataset, B: int, mp: int, mn: int) -> dict:
    """The device inputs of one impression phase, uploaded when a device route first uses it and cached on the dataset
    (as _eval_state does): users, the raw pos_num / neg_num columns, CSRs of the positive and negative lists cut to mp /
    mn (ops.list_csr; test_max_* for evaluation, train_max_* for training), the positive-history CSR (sequential models),
    and batch buffers for batches of B rows."""
    model = dataset.model
    data, corpus, dev = dataset.data, dataset.corpus, model.device
    mp, mn = int(mp), int(mn)
    st = dataset.__dict__.get("_b2r_imp")
    if st is None or st["mp"] != mp or st["mn"] != mn or st["pos_src"] is not data["pos_items"] \
            or st["neg_src"] is not data["neg_items"]:
        def up(a):
            return torch.as_tensor(np.asarray(a, dtype=np.int64)).to(dev)
        pos_ptr, pos_items = ops.list_csr(data["pos_items"], mp)
        neg_ptr, neg_items = ops.list_csr(data["neg_items"], mn)
        st = {"mp": mp, "mn": mn, "pos_src": data["pos_items"], "neg_src": data["neg_items"], "B": None,
              "users": up(data["user_id"]), "pos_num": up(data["pos_num"]), "neg_num": up(data["neg_num"]),
              "pos_ptr": up(pos_ptr), "pos_items": up(pos_items), "neg_ptr": up(neg_ptr), "neg_items": up(neg_items)}
        if hasattr(model, "history_max"):
            # ImpressionSeqModel.Dataset slices user_his[u]['pos'][:position] (BaseImpressionModel.py:206-214)
            his = {u: h["pos"] for u, h in corpus.user_his.items()}
            st["his"] = ops.DeviceHistory(his, corpus.n_users, data["user_id"], data["position"], model.history_max, dev)
            pos = np.asarray(data["position"], dtype=np.int64)
            H = int(model.history_max)
            st["lens"] = np.minimum(pos, H) if H > 0 else pos
        dataset.__dict__["_b2r_imp"] = st
    if st["B"] != B:
        bufs = {"user_id": torch.empty(B, dtype=torch.int64, device=dev),
                "item_id": torch.empty((B, mp + mn), dtype=torch.int64, device=dev)}
        if "his" in st:
            bufs["history_items"] = torch.empty(B * st["his"].width, dtype=torch.int64, device=dev)
            bufs["lengths"] = torch.empty(B, dtype=torch.int64, device=dev)
            st["widths"] = eval_history_widths(st["lens"], B)
        st["bufs"], st["B"] = bufs, B
    return st


def device_impression_batches(dataset, B: int):
    """Yields (first row, feed dict) for the batches of B rows of an impression evaluation phase (an ImpressionModel /
    ImpressionSeqModel Dataset, not under test_all), in dataset order, built on the device with the values
    collate_batch gives (models/BaseImpressionModel.py:152-184, :200-240): ``user_id``, ``item_id`` = [pos_items[:mp] |
    0-pad | neg_items[:mn] | 0-pad] (b2r_collate_impression), and for sequential models ``history_items`` / ``lengths``,
    user_his[u]['pos'][:position] cut to history_max and right-padded to the batch's longest (b2r_collate_history).
    ``pos_num`` / ``neg_num``, ``neg_history_items``, ``neg_lengths`` and the time columns are not produced: no
    kernel-backed forward reads them.  Item ids are copied exactly (the reference's float32 padding step rounds ids
    above 2^24).  Consecutive batches share the buffers: a batch must be consumed (its work enqueued on the current
    stream) before the next one is requested."""
    model = dataset.model
    B = int(B)
    st = _impression_state(dataset, B, model.test_max_pos_item, model.test_max_neg_item)
    bufs, his, users = st["bufs"], st.get("his"), st["users"]
    N = users.numel()
    for bi, start in enumerate(range(0, N, B)):
        Bn = min(B, N - start)
        ops.collate_impression(users, st["pos_ptr"], st["pos_items"], st["neg_ptr"], st["neg_items"],
                               dataset.corpus.n_users, start, Bn, st["mp"], st["mn"], bufs["user_id"], bufs["item_id"])
        feed = {"batch_size": Bn, "phase": dataset.phase, "user_id": bufs["user_id"][:Bn],
                "item_id": bufs["item_id"][:Bn]}
        if his is not None:
            hb = history_view(bufs["history_items"], Bn, st["widths"][bi])
            his.collate(users, None, start, Bn, hb, bufs["lengths"])
            feed["history_items"], feed["lengths"] = hb, bufs["lengths"][:Bn]
        yield start, feed


def impression_device_route(runner, dataset, check_sort_idx=0, all=0) -> bool:
    """Whether ImpressionRunner.evaluate (helpers/ImpressionRunner.py:135-171) can run as
    evaluate_impression_on_device: --device_metrics 1, no test_all (the reference computes no metrics there),
    neither check_sort_idx nor all (its logging and per-row returns), mn <= mp (beyond that the reference's 2 * mp wide
    label matrix raises IndexError), a pos_num column (without one :171 passes check_sort_idx as pos_num), at least one
    row, and a kernel-backed model.  Everything else keeps the reference's route."""
    model = dataset.model
    data = dataset.data
    return bool(getattr(runner, "device_metrics", 0)) and not getattr(model, "test_all", 0) \
        and check_sort_idx == 0 and all == 0 \
        and int(model.test_max_neg_item) <= int(model.test_max_pos_item) \
        and "pos_num" in data and len(data["neg_num"]) > 0 and hasattr(model, "eval_ranks")


def evaluate_impression_on_device(runner, dataset, topks: list) -> Dict[str, float]:
    """ImpressionRunner.evaluate + evaluate_method (helpers/ImpressionRunner.py:135-171, :74-133, non-test_all branch)
    with neither the inputs nor the predictions on the host: batches from device_impression_batches, the model's
    predictions of each batch ranked and scored by b2r_impression_metrics into one float64 accumulator, and the
    3 * len(topks) sums read once.  Returns NDCG@k for every k, then MAP@k, then HR@k (evaluate_method ignores
    --metric), each the float64 mean over the rows, as the reference does; the summation order differs from NumPy's,
    so values agree to about 1e-12, not bit for bit (DESIGN.md §6)."""
    model = dataset.model
    model.eval()
    ks = [int(k) for k in topks]
    # the host route's DataLoader iterator draws one int64 seed from the global CPU generator: draw it here too
    torch.empty((), dtype=torch.int64).random_()
    st = _impression_state(dataset, int(runner.eval_batch_size), model.test_max_pos_item, model.test_max_neg_item)
    acc = torch.zeros(3 * len(ks), dtype=torch.float64, device=model.device)
    fn = model.inference if hasattr(model, "inference") else model
    for start, feed in device_impression_batches(dataset, runner.eval_batch_size):
        Bn = feed["batch_size"]
        pred = fn(feed)["prediction"].contiguous()
        ops.impression_metrics(pred, st["pos_num"][start:start + Bn], st["neg_num"][start:start + Bn], st["mp"], ks, acc)
    _poll_ids(model)
    sums = acc.cpu().numpy()
    N = st["users"].numel()
    out = {}
    for m, name in enumerate(("NDCG", "MAP", "HR")):
        for i, k in enumerate(ks):
            out[f"{name}@{k}"] = np.float64(sums[m * len(ks) + i] / N)
    return out


def reference_shuffle(N: int) -> torch.Tensor:
    """The row order of one epoch of ``DataLoader(dataset, shuffle=True)`` without a generator, drawn from the global CPU
    generator exactly as torch draws it (any num_workers): ``_BaseDataLoaderIter.__init__`` takes one int64 for its
    ``_base_seed`` (torch/utils/data/dataloader.py), then ``RandomSampler.__iter__`` takes a second as the seed of a fresh
    Generator and yields ``torch.randperm(N, generator=...)`` (torch/utils/data/sampler.py).  Returns that CPU int64 [N]
    permutation and leaves the global generator where the DataLoader's epoch leaves it."""
    torch.empty((), dtype=torch.int64).random_()
    seed = int(torch.empty((), dtype=torch.int64).random_().item())
    return torch.randperm(int(N), generator=torch.Generator().manual_seed(seed))


def impression_train_device_route(runner, dataset) -> bool:
    """Whether ImpressionRunner.fit (helpers/ImpressionRunner.py:173-197) can run as fit_impression_on_device:
    --device_batches set, a kernel-backed model, pos_num and neg_num columns (the labels are built from them) and at least
    one row.  Everything else keeps the reference's route."""
    data = dataset.data
    return bool(getattr(runner, "device_batches", 0)) and hasattr(dataset.model, "eval_ranks") \
        and "pos_num" in data and "neg_num" in data and len(data["neg_num"]) > 0


def fit_impression_on_device(runner, dataset, epoch=-1) -> float:
    """ImpressionRunner.fit (helpers/ImpressionRunner.py:173-197) step for step, with the batches built on the device:
    the epoch's row order is the reference DataLoader's own (reference_shuffle, uploaded once), and per batch one
    b2r_collate_impression_train launch writes ``user_id``, ``item_id`` and the labels, and for sequential models
    b2r_collate_history the histories, right-padded to the batch's longest as collate_batch pads them.  The forward, the
    loss on those labels, backward and optimizer.step are the reference's calls, so the epoch's losses, the parameters and
    the CPU RNG state after it equal the host route's.  Each step's loss and a non-finite flag (loss or any prediction)
    stay on the device and are read once, at the end of the epoch; every flagged step logs the reference's message (which
    does not stop training).  Returns np.mean of the float32 losses, the reference's reduction.  One set of batch buffers
    serves every step: each step's work is enqueued before the next collate overwrites them."""
    model = dataset.model
    if model.optimizer is None:
        model.optimizer = runner._build_optimizer(model)
    dataset.actions_before_epoch()
    model.train()
    dev = model.device
    mp, mn, B = int(model.train_max_pos_item), int(model.train_max_neg_item), int(runner.batch_size)
    st = _impression_state(dataset, B, mp, mn)
    bufs, his, users = st["bufs"], st.get("his"), st["users"]
    if "labels" not in bufs:
        bufs["labels"] = torch.empty((B, mp + mn), dtype=torch.int64, device=dev)
    N = users.numel()
    order = reference_shuffle(N)
    perm = order.to(dev)
    widths = eval_history_widths(st["lens"][order.numpy()], B) if his is not None else None
    n_steps = (N + B - 1) // B
    losses = torch.empty(n_steps, dtype=torch.float32, device=dev)
    bad = torch.empty(n_steps, dtype=torch.bool, device=dev)
    for k, start in enumerate(range(0, N, B)):
        Bn = min(B, N - start)
        ops.collate_impression_train(users, st["pos_ptr"], st["pos_items"], st["neg_ptr"], st["neg_items"],
                                     st["pos_num"], st["neg_num"], perm, dataset.corpus.n_users, start, Bn, mp, mn,
                                     bufs["user_id"], bufs["item_id"], bufs["labels"])
        feed = {"batch_size": Bn, "phase": dataset.phase, "user_id": bufs["user_id"][:Bn],
                "item_id": bufs["item_id"][:Bn]}
        if his is not None:
            hb = history_view(bufs["history_items"], Bn, widths[k])
            his.collate(users, perm, start, Bn, hb, bufs["lengths"])
            feed["history_items"], feed["lengths"] = hb, bufs["lengths"][:Bn]
        model.optimizer.zero_grad()
        out = model(feed)
        loss = model.loss(out, bufs["labels"][:Bn])
        bad[k] = ~(torch.isfinite(loss.detach()).all() & torch.isfinite(out["prediction"].detach()).all())
        loss.backward()
        model.optimizer.step()
        losses[k] = loss.detach().reshape(())
    for _ in range(int(bad.sum())):
        logging.info("Loss is Nan. Stop training at %d." % (epoch + 1))
    out = np.mean(losses.cpu().numpy()).item()
    _poll_ids(model)
    return out


def recommend_batches(runner, dataset, k: int):
    """Yields (first row, item ids int64 [Bn, k'], scores float32 [Bn, k']) on the device for every batch of an
    evaluation phase, in dataset order: ``device_eval_batches``' batches through ``model.recommend``.  Each batch's
    tensors are its own (later batches do not overwrite them).  The out-of-range-id poll runs after the last batch."""
    model = dataset.model
    model.eval()
    start = 0
    for feed, clicked in device_eval_batches(dataset, runner.eval_batch_size):
        items, scores = model.recommend(feed, k, clicked)
        yield start, items, scores
        start += feed["batch_size"]
    _poll_ids(model)


_REC_PROBE = {"[np.int64(-3), np.float32(0.5), np.float32(1e-05)]": ops.REC_STYLE_NP,
              "[-3, 0.5, 1e-05]": ops.REC_STYLE_BARE}


def rec_csv_style(sep, users):
    """The element style (ops.REC_STYLE_NP or ops.REC_STYLE_BARE) in which ``write_rec_csv`` writes the bytes pandas
    writes for save_rec_results, or None when only pandas should write them.  The device writer needs:
      - NumPy printing scalars in one of the two styles the kernels implement: NumPy >= 2 without legacy printing
        (np.int64(3), np.float32(0.5)), or NumPy 1.x or legacy='1.25' (3, 0.5) -- decided from the version and the
        print options, and confirmed on a probe list (legacy='1.13', for one, formats float32 differently);
      - a separator that is one ASCII character other than NUL, '"', CR and LF (pandas quotes with '"' and ends lines
        with LF; any other single character only wraps the fields that contain it);
      - integer user ids that fit int64 (or none: an empty phase writes the header alone)."""
    legacy = np.get_printoptions()["legacy"]
    major = int(np.__version__.split(".")[0])
    if legacy is False:
        want = ops.REC_STYLE_NP if major >= 2 else ops.REC_STYLE_BARE
    elif legacy == "1.25":
        want = ops.REC_STYLE_BARE
    else:
        return None
    if _REC_PROBE.get(str([np.int64(-3), np.float32(0.5), np.float32(1e-05)])) != want:
        return None
    if not isinstance(sep, str) or len(sep) != 1 or not 0 < ord(sep) < 128 or sep in "\"\r\n":
        return None
    u = np.asarray(users)
    if (u.size and u.dtype.kind not in "iu") or (u.dtype == np.uint64 and u.size and int(u.max()) > np.iinfo(np.int64).max):
        return None
    return want


REC_CSV_WINDOW_BYTES = 64 << 20      # device text of one window of save_rec_results' rows (and of each pinned copy)


def _write_window(f, host: torch.Tensor, done) -> None:
    done.synchronize()               # the window's copy to the pinned buffer has landed
    f.write(memoryview(host.numpy()))


def write_rec_csv(runner, dataset, result_path: str, topk: int, sep: str, style: int) -> None:
    """save_rec_results' CSV written from the device (ops.rec_csv, include/b200rec.h): the header, then the rows of
    ``recommend_batches`` in windows of W rows, W chosen so that a window's text fits REC_CSV_WINDOW_BYTES whatever the
    phase's size.  Each batch's lists are staged into the window on the device, a full window is formatted, copied into
    one of two pinned host buffers and written with one ``write`` by a writer thread, so the file write of window i
    overlaps the lists, formatting and copy of window i + 1.  A call that fails removes the file it was writing."""
    d = os.path.dirname(result_path)
    if d:
        os.makedirs(d, exist_ok=True)
    users = _eval_state(dataset, int(runner.eval_batch_size))["users"]
    dev = users.device
    header = sep.join('"%s"' % c if sep in c else c for c in ("user_id", "rec_items", "rec_predictions")) + "\n"
    st = {"rows": 0, "filled": 0, "window": 0, "pending": [None, None]}

    def flush(ex, f):
        n = st["filled"]
        ops.rec_csv(users[st["rows"]:st["rows"] + n], st["items"][:n], st["scores"][:n], style, sep, st["text"],
                    st["offsets"])
        total = int(st["offsets"][n])
        b = st["window"] % 2
        if st["pending"][b] is not None:
            st["pending"][b].result()                               # window i - 2 is written: its buffer is free
        host = st["pinned"][b][:total]
        host.copy_(st["text"][:total], non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        st["pending"][b] = ex.submit(_write_window, f, host, done)
        st["rows"] += n
        st["filled"] = 0
        st["window"] += 1

    try:
        with open(result_path, "wb") as f, ThreadPoolExecutor(max_workers=1) as ex:
            f.write(header.encode("ascii"))
            for _, items, scores in recommend_batches(runner, dataset, topk):
                if "W" not in st:
                    kk = items.shape[1]
                    row_max = ops.rec_csv_text_bytes_max(1, kk, style)
                    W = st["W"] = max(1, min(users.numel(), REC_CSV_WINDOW_BYTES // row_max))
                    st["items"] = torch.empty((W, kk), dtype=torch.int64, device=dev)
                    st["scores"] = torch.empty((W, kk), dtype=torch.float32, device=dev)
                    st["text"] = torch.empty(W * row_max, dtype=torch.uint8, device=dev)
                    st["offsets"] = torch.empty(W + 1, dtype=torch.int64, device=dev)
                    st["pinned"] = [torch.empty(W * row_max, dtype=torch.uint8, pin_memory=True) for _ in range(2)]
                i, Bn = 0, items.shape[0]
                while i < Bn:
                    n = min(Bn - i, st["W"] - st["filled"])
                    st["items"][st["filled"]:st["filled"] + n].copy_(items[i:i + n])
                    st["scores"][st["filled"]:st["filled"] + n].copy_(scores[i:i + n])
                    st["filled"] += n
                    i += n
                    if st["filled"] == st["W"]:
                        flush(ex, f)
            if st["filled"]:
                flush(ex, f)
            for p in st["pending"]:
                if p is not None:
                    p.result()
    except BaseException:
        if os.path.exists(result_path):
            os.remove(result_path)
        raise


class BaseRunner:
    @staticmethod
    def parse_runner_args(parser):
        # helpers/BaseRunner.py:20-49 (same names, defaults and help strings' meaning)
        parser.add_argument("--epoch", type=int, default=200, help="Number of epochs.")
        parser.add_argument("--check_epoch", type=int, default=1, help="Check some tensors every check_epoch.")
        parser.add_argument("--test_epoch", type=int, default=-1, help="Print test results every test_epoch (-1: never).")
        parser.add_argument("--early_stop", type=int, default=10, help="Epochs of continuous dev drop before stopping.")
        parser.add_argument("--lr", type=float, default=1e-3, help="Learning rate.")
        parser.add_argument("--l2", type=float, default=0, help="Weight decay in optimizer.")
        parser.add_argument("--batch_size", type=int, default=256, help="Batch size during training.")
        parser.add_argument("--eval_batch_size", type=int, default=256, help="Batch size during testing.")
        parser.add_argument("--optimizer", type=str, default="Adam", help="optimizer: SGD, Adam, Adagrad, Adadelta")
        parser.add_argument("--num_workers", type=int, default=5, help="DataLoader worker processes.")
        parser.add_argument("--pin_memory", type=int, default=0, help="pin_memory in DataLoader")
        parser.add_argument("--topk", type=str, default="5,10,20,50", help="Cut-offs of the ranking metrics.")
        parser.add_argument("--metric", type=str, default="NDCG,HR", help="metrics: NDCG, HR")
        parser.add_argument("--main_metric", type=str, default="", help="Metric that selects the best model.")
        parser.add_argument("--fused_optimizer", type=int, default=0,
                            help="1: row-sparse fused SGD/Adam/Adagrad (rechorus_b200.optim) instead of torch.optim")
        parser.add_argument("--fused_step", type=int, default=0,
                            help="1 (with --fused_optimizer 1): models that offer train_step run every training step "
                                 "as one C call (forward, loss, backward, optimizer; next batch's plan prefetched)")
        parser.add_argument("--graph_step", type=int, default=0,
                            help="1 (with --fused_optimizer 1): capture the loop body of fit (zero_grad, forward, loss, "
                                 "backward, optimizer.step) once in a CUDA graph and replay it per full-size batch "
                                 "(rechorus_b200.graph.GraphedStep); the ragged last batch runs eagerly")
        parser.add_argument("--exact_adam", type=int, default=0,
                            help="1 (with --fused_optimizer 1, Adam): row-sparse cost, dense torch.optim.Adam results "
                                 "(rows are advanced through their skipped steps)")
        parser.add_argument("--device_sampler", type=int, default=0,
                            help="non-zero seed: draw the training negatives on the GPU every epoch (same distribution "
                                 "as BaseModel.py:206-214, counter-based stream)")
        parser.add_argument("--device_batches", type=int, default=0,
                            help="non-zero (a value > 1 is the seed): the whole epoch's batch production on the GPU -- "
                                 "negatives, row shuffle and collate (histories included) as device kernels "
                                 "(runner.fit_on_device); with --graph_step 1 the full-size batches replay one captured step")
        parser.add_argument("--device_metrics", type=int, default=0,
                            help="1: rank the ground truth on the GPU (model.eval_ranks) instead of copying predictions "
                                 "to the host for evaluate_method")
        return parser

    @staticmethod
    def evaluate_method(predictions: np.ndarray, topk: list, metrics: list) -> Dict[str, float]:
        """helpers/BaseRunner.py:52-78.  Column 0 holds the ground-truth item's score; its rank is the number
        of candidates scoring >= it (ties count against it)."""
        gt_rank = (predictions >= predictions[:, 0].reshape(-1, 1)).sum(axis=-1)
        out = {}
        for k in topk:
            hit = gt_rank <= k
            for metric in metrics:
                key = f"{metric}@{k}"
                if metric == "HR":
                    out[key] = hit.mean()
                elif metric == "NDCG":
                    out[key] = (hit / np.log2(gt_rank + 1)).mean()
                else:
                    raise ValueError(f"Undefined evaluation metric: {metric}.")
        return out

    def __init__(self, args):
        self.train_models = getattr(args, "train", 1)
        self.epoch = args.epoch
        self.check_epoch = args.check_epoch
        self.test_epoch = args.test_epoch
        self.early_stop = args.early_stop
        self.learning_rate = args.lr
        self.batch_size = args.batch_size
        self.eval_batch_size = args.eval_batch_size
        self.l2 = args.l2
        self.optimizer_name = args.optimizer
        self.num_workers = args.num_workers
        self.pin_memory = args.pin_memory
        self.fused_optimizer = getattr(args, "fused_optimizer", 0)
        self.device_metrics = getattr(args, "device_metrics", 0)
        self.fused_step = getattr(args, "fused_step", 0)
        self.exact_adam = getattr(args, "exact_adam", 0)
        self.graph_step = getattr(args, "graph_step", 0)
        if self.graph_step and (self.exact_adam or not self.fused_optimizer):
            raise ValueError("--graph_step 1 needs --fused_optimizer 1 and is not available with --exact_adam 1 "
                             "(the exact mode keeps per-step host bookkeeping)")
        self.device_sampler = getattr(args, "device_sampler", 0)
        self.device_batches = getattr(args, "device_batches", 0)
        self.topk = [int(x) for x in args.topk.split(",")]
        self.metrics = [m.strip().upper() for m in args.metric.split(",")]
        self.main_metric = args.main_metric or f"{self.metrics[0]}@{self.topk[0]}"
        self.main_topk = int(self.main_metric.split("@")[1]) if "@" in self.main_metric else 0
        self.time = None
        log_file = getattr(args, "log_file", "") or ""
        self.log_path = os.path.dirname(log_file)
        self.save_appendix = log_file.split("/")[-1].split(".")[0]

    def _check_time(self, start=False):
        if self.time is None or start:
            self.time = [time()] * 2
            return self.time[0]
        prev = self.time[1]
        self.time[1] = time()
        return self.time[1] - prev

    def _build_optimizer(self, model):
        logging.info("Optimizer: " + self.optimizer_name)
        if self.fused_optimizer:
            model.set_table_mode("fused")
            return RowSparseOptimizer(model, self.optimizer_name, lr=self.learning_rate, l2=self.l2,
                                      exact_dense=bool(self.exact_adam), device_clock=bool(self.graph_step))
        cls = getattr(torch.optim, self.optimizer_name)       # helpers/BaseRunner.py:112
        return cls(model.customize_parameters(), lr=self.learning_rate, weight_decay=self.l2)

    # ---------------------------------------------------------------------------------------------
    def train(self, data_dict):
        model = data_dict["train"].model
        main_results, dev_results = [], []
        self._check_time(start=True)
        try:
            for epoch in range(self.epoch):
                self._check_time()
                gc.collect()
                loss = self.fit(data_dict["train"], epoch=epoch + 1)
                if np.isnan(loss):
                    logging.info("Loss is Nan. Stop training at %d." % (epoch + 1))
                    break
                train_t = self._check_time()
                dev = self.evaluate(data_dict["dev"], [self.main_topk], self.metrics)
                dev_results.append(dev)
                main_results.append(dev[self.main_metric])
                line = "Epoch {:<5} loss={:<.4f} [{:<3.1f} s]	dev=({})".format(epoch + 1, loss, train_t,
                                                                               format_metric(dev))
                if self.test_epoch > 0 and epoch % self.test_epoch == 0:
                    test = self.evaluate(data_dict["test"], self.topk[:1], self.metrics)
                    line += " test=({})".format(format_metric(test))
                line += " [{:<.1f} s]".format(self._check_time())
                if max(main_results) == main_results[-1] or (hasattr(model, "stage") and model.stage == 1):
                    model.save_model()
                    line += " *"
                logging.info(line)
                if self.early_stop > 0 and self.eval_termination(main_results):
                    logging.info("Early stop at %d based on dev result." % (epoch + 1))
                    break
        except KeyboardInterrupt:
            logging.info("Early stop manually")
        best = main_results.index(max(main_results))
        logging.info(os.linesep + "Best Iter(dev)={:>5}\t dev=({}) [{:<.1f} s] ".format(
            best + 1, format_metric(dev_results[best]), self.time[1] - self.time[0]))
        model.load_model()

    def _fit_whole_steps(self, dataset, epoch=-1) -> float:
        """The same epoch with the loop body of helpers/BaseRunner.py:185-207 replaced by the model's single-call
        ``train_step`` (forward + loss + backward + row-sparse optimizer in one C call, the next batch's index plan
        prefetched).  Batches and RNG consumption are those of ``fit``: the per-row candidate permutation is still
        drawn (so the torch RNG stream stays in step with the reference loop) but not applied -- it is a no-op for a
        model whose candidates are scored independently, and the whole-step kernel wants the positive in column 0.
        Losses stay on the device until the epoch ends (the reference syncs on every step)."""
        model = dataset.model
        dl = DataLoader(dataset, batch_size=self.batch_size, shuffle=True, num_workers=self.num_workers,
                        collate_fn=dataset.collate_batch, pin_memory=bool(self.pin_memory))
        it = iter(dl)
        cur = next(it, None)
        cur = batch_to_device(cur, model.device) if cur is not None else None
        losses = []
        ops.bprmf_step_reset()                 # no plan prefetched by an earlier (possibly aborted) epoch survives
        try:
            while cur is not None:
                nxt = next(it, None)
                if nxt is not None:
                    nxt = batch_to_device(nxt, model.device)
                torch.rand(*cur["item_id"].shape)                     # BaseRunner.py:189's draw, see above
                same_shape = nxt is not None and nxt["item_id"].shape == cur["item_id"].shape
                losses.append(model.train_step(cur, nxt if same_shape else None))
                cur = nxt
        finally:
            ops.bprmf_step_reset()
        out = float(np.mean(torch.stack(losses).cpu().numpy())) if losses else float("nan")
        _poll_ids(model)
        return out

    def _fit_graphed(self, dataset, epoch=-1) -> float:
        """The same epoch with the loop body of helpers/BaseRunner.py:193-206 captured once in a CUDA graph
        (rechorus_b200.graph.GraphedStep) and replayed for every batch of the captured shape: one launch per step instead of
        ~70 (NeuMF) to ~150 (SASRec).  The first full-size batch trains through the capture's eager warm-up step; the ragged
        last batch runs eagerly.  As in ``_fit_whole_steps`` the per-row candidate permutation of :189 is drawn (RNG stream in
        step with the reference) but not applied: it is a no-op for candidates scored independently.  With dropout it is
        still one in distribution: every element's mask is drawn independently (keyed by its position, not by the
        candidate's identity), so permuting the candidate columns leaves the distribution of the step unchanged.  The
        dropout step counter lives on the device and advances on every replay."""
        from .graph import GraphedStep
        model = dataset.model
        dl = DataLoader(dataset, batch_size=self.batch_size, shuffle=True, num_workers=self.num_workers,
                        collate_fn=dataset.collate_batch, pin_memory=bool(self.pin_memory))
        losses = []
        for batch in dl:
            batch = batch_to_device(batch, model.device)
            torch.rand(*batch["item_id"].shape)                       # BaseRunner.py:189's draw
            gs = model.__dict__.get("_b2r_graphed_step")
            if gs is None and batch["item_id"].shape[0] == self.batch_size:
                gs = GraphedStep(model, batch, warmup=1)              # its warm-up step IS this batch's training step
                model.__dict__["_b2r_graphed_step"] = gs
                losses.append(gs.warmup_losses[0])
            elif gs is not None and gs.matches(batch):
                losses.append(gs(batch).clone())
            else:
                model.optimizer.zero_grad()
                loss = model.loss(model(batch))
                loss.backward()
                model.optimizer.step()
                losses.append(loss.detach())
        model.optimizer.sync_clock()                                  # the host step counter follows the device clock
        out = float(np.mean(torch.stack([l.reshape(()) for l in losses]).cpu().numpy())) if losses else float("nan")
        _poll_ids(model)
        return out

    def fit_on_device(self, dataset, epoch=-1) -> float:
        """SURVEY.md §8 row f3: the same epoch with BATCH PRODUCTION on the GPU (``--device_batches <seed>``).  What the
        reference does on the host -- draw the negatives (models/BaseModel.py:206-214), shuffle the rows (the
        DataLoader's RandomSampler), build one feed dict per sample and collate them (BaseModel.py:192-203,135-152) --
        becomes three device operations: ``b2r_sample_negatives`` (one Philox draw + one binary search per negative, the
        reference's distribution from a counter-based stream), a device permutation, and ``b2r_collate_general`` per
        batch.  The training step is the model's ``train_step`` (one C call) or, for models without one, the plugin
        contract's forward / loss / backward / optimizer.step on the device batch.

        Sequential datasets (models with ``history_max``, e.g. SASRec) also get ``history_items [B, Lp]`` and ``lengths
        [B]`` from ``b2r_collate_history`` (the slice of BaseModel.py:236-245 out of a device CSR of ``corpus.user_his``,
        ops.DeviceHistory).  Every batch is right-padded to the fixed width Lp = min(history_max, max position), not to
        the batch maximum as collate_batch does: the extra padding is dead work for SASRec (exact), and every full batch
        has the same shape.  ``history_times`` is not produced; no kernel-backed model reads it.

        ``--graph_step 1`` with a model without ``train_step`` (NeuMF, SASRec): the full-size batches are replayed through
        one captured step (rechorus_b200.graph.GraphedStep), each collated straight into the captured inputs just before
        its replay; the first full batch trains through the capture's warm-up step, the ragged last batch eagerly.

        RNG: the host streams of the reference are NOT reproduced (a sequential NumPy / torch CPU stream cannot be drawn
        in parallel); results are reproducible from (seed, epoch)."""
        model = dataset.model
        if model.optimizer is None:
            model.optimizer = self._build_optimizer(model)
        dev = model.device
        st = dataset.__dict__.get("_b2r_dev")
        if st is None:
            corpus = dataset.corpus
            seed = int(self.device_batches) if int(self.device_batches) > 1 else 2023
            st = {"users": torch.as_tensor(np.asarray(dataset.data["user_id"], dtype=np.int64)).to(dev),
                  "items": torch.as_tensor(np.asarray(dataset.data["item_id"], dtype=np.int64)).to(dev),
                  "sampler": ops.DeviceNegativeSampler(corpus.train_clicked_set, corpus.n_users, corpus.n_items, dev, seed=seed),
                  "gen": torch.Generator(device=dev), "seed": seed, "epoch": 0}
            if hasattr(model, "history_max"):
                st["history"] = ops.DeviceHistory(corpus.user_his, corpus.n_users, dataset.data["user_id"],
                                                  dataset.data["position"], model.history_max, dev)
            dataset.__dict__["_b2r_dev"] = st
        st["epoch"] += 1
        N, K, B = st["users"].numel(), int(model.num_neg), int(self.batch_size)
        neg = st["sampler"].sample(st["users"], K, st["epoch"])                     # [N, K] int64 on the device
        st["gen"].manual_seed(st["seed"] * 1_000_003 + st["epoch"])
        perm = torch.randperm(N, device=dev, generator=st["gen"])
        model.train()
        use_step = hasattr(model, "train_step") and isinstance(model.optimizer, RowSparseOptimizer)
        use_graph = (not use_step and bool(getattr(self, "graph_step", 0))
                     and isinstance(model.optimizer, RowSparseOptimizer))
        his = st.get("history")
        n_steps = (N + B - 1) // B
        NB = 3                                                                       # batch buffers: current, next, one being refilled

        def new_buf():
            buf = {"user_id": torch.empty(B, dtype=torch.int64, device=dev),
                   "item_id": torch.empty((B, K + 1), dtype=torch.int64, device=dev), "batch_size": B, "phase": "train"}
            if his is not None:
                buf["history_items"] = torch.empty((B, his.width), dtype=torch.int64, device=dev)
                buf["lengths"] = torch.empty(B, dtype=torch.int64, device=dev)
            return buf

        bufs = st.get("bufs")
        if bufs is None or bufs[0]["item_id"].shape != (B, K + 1):
            bufs = st["bufs"] = [new_buf() for _ in range(NB)]

        def fill(buf, k, Bn):
            # two launches: user / candidate columns, then (sequential models) the history
            ops.collate_general(st["users"], st["items"], neg, perm, k * B, Bn, buf["user_id"], buf["item_id"])
            if his is not None:
                his.collate(st["users"], perm, k * B, Bn, buf["history_items"], buf["lengths"])

        def batch(k):
            Bn = min(B, N - k * B)
            buf = bufs[k % NB]
            fill(buf, k, Bn)
            if Bn == B:
                return buf
            out = {key: (v[:Bn] if isinstance(v, torch.Tensor) else v) for key, v in buf.items()}
            out["batch_size"] = Bn
            return out

        def eager_step(feed):
            model.optimizer.zero_grad()
            loss = model.loss(model(feed))
            loss.backward()
            model.optimizer.step()
            return loss.detach()

        losses = []
        ops.bprmf_step_reset()
        try:
            if use_graph:
                from .graph import GraphedStep
                gs = model.__dict__.get("_b2r_graphed_step")
                for k in range(n_steps):
                    if N - k * B < B:
                        losses.append(eager_step(batch(k)))                         # the ragged last batch
                    elif gs is None or not gs.matches(bufs[0]):
                        gs = GraphedStep(model, batch(k), warmup=1)                 # its warm-up step IS this batch's step
                        model.__dict__["_b2r_graphed_step"] = gs
                        losses.append(gs.warmup_losses[0])
                    else:
                        # straight into the captured inputs; on the same stream, so after the previous replay read them
                        fill(gs.static, k, B)
                        losses.append(gs.replay().clone())
                model.optimizer.sync_clock()                                       # the host step counter follows the device clock
            else:
                cur = batch(0)
                for k in range(n_steps):
                    nxt = batch(k + 1) if k + 1 < n_steps else None
                    if use_step:
                        same = nxt is not None and nxt["item_id"].shape == cur["item_id"].shape
                        losses.append(model.train_step(cur, nxt if same else None))
                    else:
                        losses.append(eager_step(cur))
                    cur = nxt
        finally:
            ops.bprmf_step_reset()
        out = float(torch.stack(losses).mean().cpu()) if losses else float("nan")
        _poll_ids(model)
        return out

    def fit(self, dataset, epoch=-1) -> float:
        """helpers/BaseRunner.py:174-208, step for step."""
        model = dataset.model
        opt = model.optimizer
        if opt is None or (self.graph_step and isinstance(opt, RowSparseOptimizer) and not opt._want_clock and opt.t == 0):
            model.optimizer = self._build_optimizer(model)     # (a lazily built one without the device clock is replaced)
        if self.device_sampler and model.__dict__.get("_b2r_device_sampler") is None:
            corpus = dataset.corpus
            model.__dict__["_b2r_device_sampler"] = ops.DeviceNegativeSampler(
                corpus.train_clicked_set, corpus.n_users, corpus.n_items, model.device, seed=self.device_sampler)
        if self.device_batches:
            return self.fit_on_device(dataset, epoch)
        dataset.actions_before_epoch()
        model.train()
        if self.fused_step and hasattr(model, "train_step") and isinstance(model.optimizer, RowSparseOptimizer):
            return self._fit_whole_steps(dataset, epoch)
        if self.graph_step and isinstance(model.optimizer, RowSparseOptimizer):
            return self._fit_graphed(dataset, epoch)
        losses = []
        dl = DataLoader(dataset, batch_size=self.batch_size, shuffle=True, num_workers=self.num_workers,
                        collate_fn=dataset.collate_batch, pin_memory=bool(self.pin_memory))
        for batch in dl:
            batch = batch_to_device(batch, model.device)
            item_ids = batch["item_id"]
            # per-row candidate permutation drawn from the CPU generator, as the reference does (:189)
            indices = torch.argsort(torch.rand(*item_ids.shape), dim=-1)
            rows = torch.arange(item_ids.shape[0]).unsqueeze(-1)
            batch["item_id"] = item_ids[rows, indices]
            model.optimizer.zero_grad()
            out = model(batch)
            pred = out["prediction"]
            if pred.dim() == 2:
                restored = torch.zeros(*pred.shape).to(pred.device)
                restored[rows, indices] = pred                           # autograd-tracked index_put (:201)
                out["prediction"] = restored
            loss = model.loss(out)
            loss.backward()
            model.optimizer.step()
            losses.append(loss.detach().cpu().data.numpy())
        _poll_ids(model)
        return float(np.mean(losses))

    def eval_termination(self, criterion: List[float]) -> bool:
        """helpers/BaseRunner.py:132-137 with utils.non_increasing (utils/utils.py:103-104): stop when the FIRST value
        of the last ``early_stop`` results is >= every later one of that window (not a pairwise-monotone test), or when
        the best result is more than ``early_stop`` epochs old."""
        if len(criterion) > self.early_stop:
            w = criterion[-self.early_stop:]
            if all(w[0] >= y for y in w[1:]):
                return True
        return len(criterion) - criterion.index(max(criterion)) > self.early_stop

    def evaluate(self, dataset, topks: list, metrics: list) -> Dict[str, float]:
        if self.device_metrics and hasattr(dataset.model, "eval_ranks"):
            return self.evaluate_on_device(dataset, topks, metrics)
        return self.evaluate_method(self.predict(dataset), topks, metrics)

    def evaluate_on_device(self, dataset, topks: list, metrics: list) -> Dict[str, float]:
        """helpers/BaseRunner.py:216-252 with neither the inputs nor the predictions on the host: the batches come from
        ``device_eval_batches`` (no DataLoader, no feed dicts), per batch the model returns the integer ranks of the
        ground truth (``eval_ranks``; under test_all masked from the clicked-item CSR), a rank histogram is accumulated
        on the device and HR@k / NDCG@k are read off it -- (max k + 2) integers cross PCIe per evaluation, and the
        histogram read and the id poll are the only synchronisations."""
        model = dataset.model
        model.eval()
        kmax = max(int(k) for k in topks)
        # the host route's DataLoader iterator draws one int64 seed from the global CPU generator: draw it here too, so the
        # training epochs that follow an evaluation shuffle their rows as the reference's run does
        torch.empty((), dtype=torch.int64).random_()
        hist = torch.zeros(kmax + 2, dtype=torch.int64, device=model.device)
        n_rows = 0
        for feed, clicked in device_eval_batches(dataset, self.eval_batch_size):
            hist += ops.rank_histogram(model.eval_ranks(feed, clicked=clicked), kmax)
            n_rows += feed["batch_size"]
        _poll_ids(model)
        return ops.metrics_from_histogram(hist, n_rows, topks, metrics)

    def predict(self, dataset, save_prediction: bool = False) -> np.ndarray:
        """helpers/BaseRunner.py:225-252 (uses the model's no-grad ``inference`` hook when present)."""
        model = dataset.model
        model.eval()
        preds = []
        dl = DataLoader(dataset, batch_size=self.eval_batch_size, shuffle=False, num_workers=self.num_workers,
                        collate_fn=dataset.collate_batch, pin_memory=bool(self.pin_memory))
        for batch in dl:
            batch = batch_to_device(batch, model.device)
            fn = model.inference if hasattr(model, "inference") else model
            preds.extend(fn(batch)["prediction"].cpu().data.numpy())
        _poll_ids(model)
        preds = np.array(preds)
        if model.test_all:
            rows, cols = [], []
            for i, u in enumerate(dataset.data["user_id"]):
                clicked = list(dataset.corpus.train_clicked_set[u] | dataset.corpus.residual_clicked_set[u])
                rows.extend([i] * len(clicked))
                cols.extend(clicked)
            preds[rows, cols] = -np.inf
        return preds

    def recommend(self, dataset, k: int = 100):
        """The top-k' recommendation list of every row of an evaluation phase (main.py:117-132's TopK branch) computed on
        the device: (users as dataset.data["user_id"] holds them, item ids int64 [N, k'], scores float32 [N, k']) as host
        arrays, rows in dataset order.  The batches are evaluate_on_device's (``device_eval_batches``); under test_all a
        dot-product model scores the catalogue itself (ops.topk_all_items) and NeuMF's [target | arange(1, n_items)]
        predictions are masked with ops.mask_clicked."""
        out_items, out_scores = [], []
        for _, items, scores in recommend_batches(self, dataset, k):
            out_items.append(items)
            out_scores.append(scores)
        if not out_items:
            return list(dataset.data["user_id"]), np.zeros((0, 0), np.int64), np.zeros((0, 0), np.float32)
        return (list(dataset.data["user_id"]), torch.cat(out_items).cpu().numpy(), torch.cat(out_scores).cpu().numpy())

    def save_rec_results(self, dataset, result_path: str, topk: int = 100, sep: str = "\t") -> None:
        """The TopK branch of main.py:117-132 (save_rec_results) with the lists from ``recommend``: the CSV matches the
        reference's byte for byte.  When ``rec_csv_style`` says the device can write what pandas writes, the lists never
        leave the device: ``write_rec_csv`` formats them there, window by window.  Otherwise the lists are written as the
        reference writes them, a DataFrame of Python lists of NumPy scalars through pandas' to_csv."""
        style = rec_csv_style(sep, dataset.data["user_id"])
        if style is not None:
            write_rec_csv(self, dataset, result_path, topk, sep, style)
            return
        import pandas as pd
        users, items, scores = self.recommend(dataset, topk)
        d = os.path.dirname(result_path)
        if d:
            os.makedirs(d, exist_ok=True)
        rec_df = pd.DataFrame(columns=["user_id", "rec_items", "rec_predictions"])
        rec_df["user_id"] = users
        rec_df["rec_items"] = [list(r) for r in items]
        rec_df["rec_predictions"] = [list(r) for r in scores]
        rec_df.to_csv(result_path, sep=sep, index=False)

    def print_res(self, dataset) -> str:
        return "(" + format_metric(self.evaluate(dataset, self.topk, self.metrics)) + ")"
