"""The impression setting end to end on an H100: the reference's UNCHANGED ``src/main.py`` (the copy build() stages in
oracle/_ref/src) runs BPRMFImpression and SASRecImpression through ``rechorus_b200.overlay`` on a tiny impression dataset,
once with the reference's ImpressionRunner.evaluate and once with ``--device_metrics 1`` (B200ImpressionRunner).  Training
is the same code on the same seeds in both runs, and the device route draws the host route's one CPU-generator seed per
evaluation, so the epoch losses are identical; every dev / test metric line is identical too.  Skipped only where
build() had no reference to stage."""
import os
import re
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "src")          # oracle/stage_reference.py

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "main.py")),
                                 reason="no unmodified reference staged in oracle/_ref (build() without the checkout)")]

N_USERS, N_ITEMS, PER_USER = 30, 80, 6


def _dataset(root):
    """impressions of 1-5 clicked and 1-7 skipped items per (user, time); per user the first impressions train, the
    last two are dev and test"""
    rng = np.random.RandomState(3)
    d = os.path.join(root, "data", "tiny_imp")
    os.makedirs(d)
    parts = {"train": [], "dev": [], "test": []}
    t = 0
    for u in range(1, N_USERS):
        for j in range(PER_USER):
            t += 1
            phase = "train" if j < PER_USER - 2 else ("dev" if j == PER_USER - 2 else "test")
            items = rng.choice(np.arange(1, N_ITEMS), rng.randint(2, 13), replace=False)
            npos = rng.randint(1, min(5, len(items) - 1) + 1)
            for k, i in enumerate(items):
                parts[phase].append((u, int(i), t, int(k < npos)))
    for phase, rows in parts.items():
        pd.DataFrame(rows, columns=["user_id", "item_id", "time", "label"]).to_csv(
            os.path.join(d, phase + ".csv"), sep="\t", index=False)
    return os.path.join(root, "data") + "/"


def _run(tmp, tag, model, extra):
    cwd = os.path.join(tmp, tag, "src")
    os.makedirs(cwd)
    cmd = [sys.executable, "-m", "rechorus_b200.overlay", "--ref", REF, "--model_name", model, "--model_mode", "Impression",
           "--dataset", "tiny_imp", "--path", os.path.join(tmp, "data") + "/", "--gpu", "0", "--num_workers", "0",
           "--epoch", "2", "--early_stop", "0", "--test_epoch", "1", "--batch_size", "16", "--eval_batch_size", "7",
           "--emb_size", "16", "--lr", "0.01", "--l2", "0", "--topk", "1,3,5", "--metric", "NDCG,HR",
           "--impression_idkey", "time", "--train_max_pos_item", "4", "--train_max_neg_item", "4",
           "--test_max_pos_item", "4", "--test_max_neg_item", "3", "--model_path", os.path.join(tmp, tag, "model.pt"),
           "--log_file", os.path.join(tmp, tag, "log.txt"), "--regenerate", "1", "--save_final_results", "0", *extra]
    res = subprocess.run(cmd, cwd=cwd, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=900)
    out = res.stdout + res.stderr
    assert res.returncode == 0, out[-3000:]
    losses = re.findall(r"Epoch \d+\s+loss=([0-9.]+)", out)
    metric_lines = re.findall(r"(?:dev|test)=\(([^)]*)\)", out) + re.findall(r"Training: \(([^)]*)\)", out)
    return losses, metric_lines, out


@pytest.mark.parametrize("model,extra", [("BPRMF", []),
                                         ("SASRec", ["--history_max", "5", "--num_layers", "1", "--num_heads", "1"])])
def test_device_metrics_reproduces_the_reference_evaluate(tmp_path, model, extra):
    tmp = str(tmp_path)
    _dataset(tmp)
    host_l, host_m, host_out = _run(tmp, "host", model, extra)
    dev_l, dev_m, dev_out = _run(tmp, "device", model, [*extra, "--device_metrics", "1"])
    # main.py's argument table lists --device_metrics only when the runner's parser knows it (B200ImpressionRunner)
    assert re.search(r"device_metrics\s*\|\s*1", dev_out) and not re.search(r"device_metrics\s*\|", host_out)
    assert len(host_l) == 2 and dev_l == host_l
    assert len(host_m) >= 6 and dev_m == host_m
    assert any("MAP@3" in m for m in host_m)
