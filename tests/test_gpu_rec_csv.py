"""GPU: save_rec_results' CSV written on the device (b2r_rec_csv, runner.write_rec_csv) against its two references:

  - the formatter inside the kernels equals the host harness (tests/rec_format_harness.cu, pinned against NumPy by
    tests/test_rec_csv_cpu.py) bit for bit, on the designed sample and 2^26 random float32 patterns;
  - save_rec_results' bytes equal what pandas writes for the same ``recommend`` lists (the writer isolated, so the
    comparison is exact for every model): BPRMF, NeuMF and SASRec with and without test_all, the separators a user
    passes, both element styles, windows that split batches, k beyond the candidate count, an empty phase, and scores
    holding -inf, NaN, -0.0 and subnormals;
  - the fallbacks (other NumPy printing, a multi-character separator) still go through pandas, and two runs write
    identical files."""
import argparse
import os
import sys

import numpy as np
import pandas as pd
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from tests import rec_csv_oracle as O  # noqa: E402

pytestmark = [pytest.mark.gpu]
DEV = torch.device("cuda", 0)


# ---- the device formatter ----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return O.build_harness(str(tmp_path_factory.mktemp("rec_harness")))


def _device_rows(users, items, scores, style, sep="\t"):
    from rechorus_b200 import ops
    N, k = items.shape
    out = torch.empty(ops.rec_csv_text_bytes_max(N, k, style), dtype=torch.uint8, device=DEV)
    offs = torch.empty(N + 1, dtype=torch.int64, device=DEV)
    ops.rec_csv(torch.from_numpy(users).to(DEV), torch.from_numpy(items).to(DEV),
                torch.from_numpy(scores.view(np.float32)).to(DEV), style, sep, out, offs)
    offs = offs.cpu().numpy()
    return out[:int(offs[N])].cpu().numpy().tobytes(), offs


@pytest.mark.parametrize("what", ["designed_np", "designed_bare", "random_np"])
def test_device_formatter_equals_the_host_harness(exe, tmp_path, what):
    """rows of k = 1024 elements; scores are the patterns under test, items cycle through the int64 edge sample"""
    style = O.STYLE_BARE if what.endswith("bare") else O.STYLE_NP
    if what.startswith("designed"):
        bits = O.designed_sample()
    else:
        bits = np.random.RandomState(5).randint(0, 1 << 32, 1 << 26, dtype=np.uint64).astype(np.uint32)
    ints = O.int64_sample()
    int_text = O.harness(exe, ints, style, str(tmp_path), ints=True, raw=True)
    k, chunk = 1024, 1 << 22
    for lo in range(0, bits.size, chunk):
        b = bits[lo:lo + chunk]
        N = -(-b.size // k)
        b = np.concatenate([b, np.zeros(N * k - b.size, np.uint32)])         # the last row padded with +0.0
        idx = np.arange(lo, lo + N * k) % ints.size
        users = np.arange(lo, lo + N, dtype=np.int64)
        got, offs = _device_rows(users, ints[idx].reshape(N, k), b.reshape(N, k), style)
        ft = O.harness(exe, b, style, str(tmp_path), raw=True)
        it = [int_text[i] for i in idx]
        uid = O.harness(exe, users, O.STYLE_BARE, str(tmp_path), ints=True, raw=True)
        rows = [b"%s\t[%s]\t[%s]\n" % (uid[r], b", ".join(it[r * k:(r + 1) * k]), b", ".join(ft[r * k:(r + 1) * k]))
                for r in range(N)]
        assert np.array_equal(np.diff(offs), [len(r) for r in rows])
        if got != b"".join(rows):
            want = b"".join(rows)
            at = next(i for i in range(min(len(got), len(want))) if got[i] != want[i])
            raise AssertionError((lo, got[max(0, at - 80):at + 80], want[max(0, at - 80):at + 80]))


def test_quoting_follows_each_field():
    """a field is quoted exactly when it contains sep: per row, per cell"""
    users = np.array([1, 10, 2, -3], dtype=np.int64)
    items = np.array([[5, 6], [7, 8], [9, 10], [11, 12]], dtype=np.int64)
    scores = np.array([[0.5, 1e-05], [2.5, 3.5], [np.inf, -np.inf], [np.nan, -0.0]], dtype=np.float32)
    for sep in ("1", "e", "-", ",", " ", "[", "\t", "n", "5"):
        want = pd.DataFrame({"user_id": users, "rec_items": [list(r) for r in items],
                             "rec_predictions": [list(r) for r in scores]}).to_csv(sep=sep, index=False)
        got, _ = _device_rows(users, items, scores, O.STYLE_NP, sep)
        assert got.decode() == want.split("\n", 1)[1], sep


# ---- save_rec_results --------------------------------------------------------------------------------------------

MODELS = {
    "BPRMF": ["--emb_size", "64"],
    "NeuMF": ["--emb_size", "32", "--layers", "[32, 16]"],
    "SASRec": ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "8"],
}


def _setup(name, test_all, rows=None):
    import fit_corpus
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    p = cls.parse_model_args(p)
    a = p.parse_args([*MODELS[name], "--num_workers", "0", "--eval_batch_size", "16", "--test_all", str(test_all)])
    a.device, a.model_path, a.log_file = DEV, "/tmp/_b2r_rec_csv.pt", ""
    corpus = fit_corpus.build()
    if rows is not None:
        corpus.data_df["test"] = corpus.data_df["test"].iloc[:rows]
    torch.manual_seed(0)
    model = cls(a, corpus).to(DEV)
    with torch.no_grad():
        for prm in model.parameters():
            prm.mul_(30.0)
    ds = cls.Dataset(model, corpus, "test")
    ds.prepare()
    return model, ds, BaseRunner(a)


SPECIALS = np.array([0xff800000, 0x7fc00000, 0x80000000, 0x00000001, 0x807fffff, 0x00400000, 0xffc00001, 0x7f800000,
                     0x3727c5ac, 0x5a0e1bca, 0x49742400, 0x38d1b717], dtype=np.uint32).view(np.float32)


def _plant_specials(model):
    """model.recommend with the first scores of every batch replaced by -inf, NaNs, -0.0, subnormals, inf and values at
    the notation switch points"""
    orig = model.recommend
    sp = torch.from_numpy(SPECIALS.copy()).to(DEV)

    def recommend(feed, k, clicked=None):
        items, scores = orig(feed, k, clicked)
        scores = scores.clone()
        n = min(scores.numel(), sp.numel())
        scores.view(-1)[:n] = sp[:n]
        return items, scores
    model.recommend = recommend


def _check(tmp_path, model, ds, runner, k, sep, tag, device_route=True):
    users, items, scores = runner.recommend(ds, k)
    want = O.pandas_csv(str(tmp_path / f"{tag}-pandas.csv"), users, items, scores, sep)
    path = str(tmp_path / "out" / f"{tag}.csv")
    if device_route:
        def refuse(*a, **kw):
            raise AssertionError("the pandas writer ran")
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(pd.DataFrame, "to_csv", refuse)
            runner.save_rec_results(ds, path, k, sep=sep)
    else:
        runner.save_rec_results(ds, path, k, sep=sep)
    with open(path, "rb") as f:
        got = f.read()
    assert got == want, (got[:400], want[:400])
    return got


@pytest.mark.parametrize("name", ["BPRMF", "NeuMF", "SASRec"])
@pytest.mark.parametrize("test_all", [0, 1])
def test_save_rec_results_equals_pandas_on_the_same_lists(tmp_path, name, test_all):
    model, ds, runner = _setup(name, test_all)
    for k in (10, 100):                                    # 100 is more than the candidates (20, or 50 under test_all)
        _check(tmp_path, model, ds, runner, k, "\t", f"{name}{test_all}-{k}")


@pytest.mark.parametrize("legacy", [False, "1.25"])
def test_separators_styles_specials_and_split_windows(tmp_path, monkeypatch, legacy):
    from rechorus_b200 import runner as R
    model, ds, runner = _setup("BPRMF", 1)
    _plant_specials(model)
    with np.printoptions(legacy=legacy):
        for cap in (R.REC_CSV_WINDOW_BYTES, 7000, 20000):   # 2 to 9 rows per window: windows split batches of 16
            monkeypatch.setattr(R, "REC_CSV_WINDOW_BYTES", cap)
            for sep in ("\t", ",", " ", ";", "1", "e"):
                _check(tmp_path, model, ds, runner, 100, sep, f"{legacy}-{cap}-{ord(sep)}")


def test_empty_phase_writes_the_header(tmp_path):
    model, ds, runner = _setup("BPRMF", 1, rows=0)
    assert len(ds) == 0
    for sep in ("\t", "e"):
        path = str(tmp_path / f"empty{ord(sep)}.csv")
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(pd.DataFrame, "to_csv", lambda *a, **kw: pytest.fail("the pandas writer ran"))
            runner.save_rec_results(ds, path, 100, sep=sep)
        want = O.pandas_csv(str(tmp_path / "want.csv"), [], np.zeros((0, 0), np.int64), np.zeros((0, 0), np.float32), sep)
        assert open(path, "rb").read() == want


def test_fallbacks_go_through_pandas(tmp_path):
    model, ds, runner = _setup("NeuMF", 0)
    with np.printoptions(legacy="1.13"):
        _check(tmp_path, model, ds, runner, 100, "\t", "legacy113", device_route=False)
    with pytest.raises(TypeError):                          # pandas' own error for a multi-character separator
        runner.save_rec_results(ds, str(tmp_path / "bad.csv"), 100, sep="::")


def test_two_runs_write_identical_files(tmp_path, monkeypatch):
    from rechorus_b200 import runner as R
    monkeypatch.setattr(R, "REC_CSV_WINDOW_BYTES", 50000)
    model, ds, runner = _setup("SASRec", 0)
    paths = [str(tmp_path / f"run{i}.csv") for i in range(2)]
    for p in paths:
        runner.save_rec_results(ds, p, 100, sep="\t")
    a, b = (open(p, "rb").read() for p in paths)
    assert a == b and a.count(b"\n") == len(ds) + 1
