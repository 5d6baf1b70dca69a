"""CPU: the dropout mask definition (tests/dropout_oracle.py, the restatement of b2r_dropout) against the fixtures the
reference's own NeuMF / SASRec produced with it (tests/golden/make_dropout_golden.py), its statistics, and the model-side
host logic (seed without drawing, validation, state_dict keys)."""
import argparse
import ast
import os
import types

import numpy as np
import pytest
import torch

from oracle import rechorus_oracle as O
from tests import dropout_oracle as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    meta = ast.literal_eval(str(z["meta"]))
    pick = lambda pre: {k[len(pre):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(pre)}  # noqa: E731
    return meta, z, pick("w:"), pick("in:"), pick("g:")


def test_vectorised_philox_equals_the_oracle():
    rng = np.random.RandomState(0)
    for _ in range(20):
        ctr = [int(v) for v in rng.randint(0, 2 ** 32, 4, dtype=np.uint64)]
        key = [int(v) for v in rng.randint(0, 2 ** 32, 2, dtype=np.uint64)]
        got = [int(w[0]) for w in D.philox4x32_10_np(*[np.array([c], dtype=np.uint64) for c in ctr], *key)]
        assert got == O.philox4x32_10(ctr, key)


def test_oracle_reproduces_every_fixture_mask():
    meta, z, _, batch, _ = _load("neumf_dropout")
    B, C = meta["B"], meta["C"]
    for l, w in enumerate(meta["layers"]):
        assert np.array_equal(z[f"mask:{l}"].reshape(B * C, w), D.neumf_mask(meta["seed"], meta["step"], l, B, C, w, meta["p"]))
    meta, z, _, batch, _ = _load("sasrec_dropout")
    B, Lb = batch["history_items"].shape
    for site in range(2 * meta["num_layers"]):
        assert np.array_equal(z[f"mask:{site}"], D.sasrec_mask(meta["seed"], meta["step"], site, B, Lb, meta["d"], meta["p"]))


@pytest.mark.parametrize("model_name,fixture", [("NeuMF", "neumf_dropout"), ("SASRec", "sasrec_dropout")])
def test_oracle_with_fixture_masks_reproduces_reference(model_name, fixture):
    meta, z, w, batch, g_ref = _load(fixture)
    masks = {int(k[5:]): torch.from_numpy(z[k]) for k in z.files if k.startswith("mask:")}
    s = D.dropout_scale(meta["p"])
    pred, loss, grads = D.loss_and_grads(model_name, w, batch, masks, s, meta.get("num_heads", 4))
    assert (pred - torch.from_numpy(z["prediction"])).abs().max() <= 1e-5
    assert abs(float(loss) - float(z["loss"])) <= 1e-5
    for k in g_ref:
        assert (grads[k] - g_ref[k]).abs().max() <= 1e-5, k


def test_sasrec_fixture_padding_is_invariant():
    meta, z, w, batch, g_ref = _load("sasrec_dropout")
    assert (torch.from_numpy(z["pad:prediction"]) - torch.from_numpy(z["prediction"])).abs().max() <= 1e-6
    for k in g_ref:
        assert (torch.from_numpy(z["pad:g:" + k]) - g_ref[k]).abs().max() <= 1e-6, k


@pytest.mark.parametrize("p", [0.1, 0.2, 0.5])
def test_keep_fraction_and_independence(p):
    n_rows, w = 8192, 128                                     # 2^20 elements per mask
    masks = {(site, step): D.dropout_mask(12345, step, site, np.arange(n_rows), np.arange(n_rows) % 50, w, p)
             for site, step in [(0, 0), (1, 0), (0, 1)]}
    n = n_rows * w
    for m in masks.values():
        sigma = np.sqrt(p * (1 - p) / n)
        assert abs(m.mean() - (1 - p)) <= 5 * sigma
    agree = (1 - p) ** 2 + p ** 2
    sigma = np.sqrt(agree * (1 - agree) / n)
    for other in [(1, 0), (0, 1)]:
        rate = (masks[(0, 0)] == masks[other]).mean()
        assert abs(rate - agree) <= 5 * sigma, (other, rate, agree)


def test_mask_edges():
    assert D.dropout_mask(1, 0, 0, np.arange(64), np.zeros(64), 20, 1.0).sum() == 0
    assert D.dropout_mask(1, 0, 0, np.arange(64), np.zeros(64), 20, 0.0).all()
    assert D.dropout_scale(1.0) == 0.0 and D.dropout_scale(0.2) == 1.25


def _model(name, dropout):
    from rechorus_b200 import plugin
    cls = getattr(plugin, name)
    a = cls.parse_model_args(argparse.ArgumentParser()).parse_args(["--emb_size", "16", "--dropout", str(dropout)])
    a.device, a.model_path = torch.device("cpu"), "/tmp/_b2r_unused.pt"
    return cls(a, types.SimpleNamespace(n_users=20, n_items=30))


@pytest.mark.parametrize("name", ["NeuMF", "SASRec"])
def test_building_a_dropout_model_draws_nothing_extra(name):
    draws = []
    for p in (0.0, 0.2):
        torch.manual_seed(42)
        np.random.seed(42)
        m = _model(name, p)
        draws.append((torch.rand(8), np.random.rand(4), sorted(m.state_dict())))
    assert torch.equal(draws[0][0], draws[1][0]) and np.array_equal(draws[0][1], draws[1][1])
    assert draws[0][2] == draws[1][2]                          # no dropout state in the state_dict


@pytest.mark.parametrize("name", ["NeuMF", "SASRec"])
def test_dropout_outside_unit_interval_is_rejected(name):
    with pytest.raises(ValueError):
        _model(name, 1.5)
