#!/usr/bin/env python
"""Time of one impression training epoch (``fit(train, epoch)``) on the device route (B200ImpressionRunner with
--device_batches 1: the reference DataLoader's row order, b2r_collate_impression_train batches and labels, losses read once
per epoch) and on the host route (the reference's own ImpressionRunner.fit from the copy build() stages in oracle/_ref:
DataLoader with 5 workers, one feed dict per impression, collate_batch, host-to-device copies, labels from pos_num /
neg_num, and the per-step synchronisations of its NaN check and loss read):

  bprmf    BPRMFImpression, d = 64
  sasrec   SASRecImpression, d = 64, 1 block, 1 head, history_max 20

on 200,000 training impressions with train_max_pos_item = train_max_neg_item = 20 (lists of 1-25 positives and 1-25
negatives), batch 256, Adam, loss BPR.  Each route trains its own identically initialised model (the overlay's classes, as
main.py runs them) for 2 epochs from the same CPU seed; each epoch is timed with CUDA events around the call followed by
torch.cuda.synchronize().  The device route's first epoch also uploads the set's lists.  The two routes' epoch losses are
reported side by side (the device route reproduces the host route's batches, so they are equal).  Without a staged
reference only the device route is timed, on the stand-alone plugin classes, and the output says so.  One JSON line per
case, then one with the card's name, power limit and max SM clock read in the same run.

    python tools/impression_fit_time.py [--epochs 2] [--num_workers 5] [--cases bprmf sasrec]
"""
import argparse
import json
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
REF = os.path.join(ROOT, "oracle", "_ref", "src")

N_ROWS, N_USERS, N_ITEMS, MP, MN, BS, HIS = 200_000, 50_000, 100_000, 20, 20, 256, 30
CASES = {"bprmf": ("BPRMFImpression", ["--emb_size", "64"]),
         "sasrec": ("SASRecImpression", ["--emb_size", "64", "--num_layers", "1", "--num_heads", "1", "--history_max", "20"])}
OVERLAY_CLASSES = {}                                              # overlay.install's classes, when a reference is staged


def corpus(seed=0):
    """a training set of N_ROWS impressions as ImpressionReader / ImpressionSeqReader leave it and user_his with HIS
    positives / 5 negatives per user"""
    from impression_eval_time import corpus as eval_corpus
    c = eval_corpus(seed)
    c.data_df = {"train": c.data_df["dev"]}
    return c


def timed(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / 1e3, out


def have_reference() -> bool:
    return os.path.isfile(os.path.join(REF, "main.py"))


def model_and_dataset(name, c):
    cls_name, flags = CASES[name]
    flags = flags + ["--train_max_pos_item", str(MP), "--train_max_neg_item", str(MN), "--loss_n", "BPR"]
    if have_reference():
        import models.BaseImpressionModel as RI
        cls = OVERLAY_CLASSES[cls_name]
        ds_cls = RI.ImpressionSeqModel.Dataset if "SASRec" in cls_name else RI.ImpressionModel.Dataset
    else:
        from rechorus_b200 import plugin
        cls, ds_cls = getattr(plugin, cls_name), None
    a = cls.parse_model_args(argparse.ArgumentParser()).parse_args(flags)
    a.device, a.model_path = torch.device("cuda", 0), "/tmp/_b2r_imp_fit_time.pt"
    torch.manual_seed(0)
    model = cls(a, c).to(a.device)
    if ds_cls is not None:
        return model, ds_cls(model, c, "train")
    data = c.data_df["train"].to_dict("list")
    return model, types.SimpleNamespace(model=model, corpus=c, data=data, phase="train",
                                        actions_before_epoch=lambda: None)


def run_case(name, epochs, num_workers, c):
    from rechorus_b200.runner import fit_impression_on_device
    out = {"case": name, "model": CASES[name][0], "rows": N_ROWS, "mp": MP, "mn": MN, "batch_size": BS,
           "epochs": epochs}
    ra = argparse.Namespace(epoch=epochs, check_epoch=1, test_epoch=-1, early_stop=0, lr=1e-3, l2=0.0, batch_size=BS,
                            eval_batch_size=BS, optimizer="Adam", num_workers=num_workers, pin_memory=0, topk="5",
                            metric="NDCG", main_metric="", train=1, log_file="", device_batches=1)
    routes = {}
    if have_reference():
        from helpers.ImpressionRunner import ImpressionRunner

        from rechorus_b200 import overlay
        routes["host"] = ImpressionRunner(ra)
        routes["device"] = overlay._make_impression_runner_module(ImpressionRunner).B200ImpressionRunner(ra)
    else:
        from rechorus_b200.runner import BaseRunner
        dev = BaseRunner(ra)
        routes["device"] = types.SimpleNamespace(fit=lambda ds, e: fit_impression_on_device(dev, ds, e))
        out["host"] = "not measured: no reference staged in oracle/_ref"
    for route, runner in routes.items():
        model, ds = model_and_dataset(name, c)
        torch.manual_seed(1)
        times, losses = [], []
        for e in range(1, epochs + 1):
            t, loss = timed(lambda: runner.fit(ds, e))
            times.append(round(t, 3))
            losses.append(loss)
        out[f"{route}_epoch_s"], out[f"{route}_losses"] = times, losses
        del model, ds
        torch.cuda.empty_cache()
    if "host" in routes:
        out["num_workers"] = num_workers
        out["host_over_device_last_epoch"] = round(out["host_epoch_s"][-1] / out["device_epoch_s"][-1], 1)
        out["same_losses"] = out["host_losses"] == out["device_losses"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--num_workers", type=int, default=5, help="the host route's DataLoader workers (runner default 5)")
    ap.add_argument("--cases", nargs="*", default=list(CASES))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("impression_fit_time.py measures on a CUDA device; none found")
    if have_reference():
        from rechorus_b200 import overlay
        OVERLAY_CLASSES.update(overlay.install(REF))
    else:
        print("no reference staged in oracle/_ref: timing the device route only", flush=True)
    from seq_batches_time import card
    c = corpus()
    for name in a.cases:
        print(json.dumps(run_case(name, a.epochs, a.num_workers, c)), flush=True)
    print(json.dumps(card()), flush=True)


if __name__ == "__main__":
    main()
