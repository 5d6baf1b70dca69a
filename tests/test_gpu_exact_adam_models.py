"""GPU tests of the exact dense-Adam mode (RowSparseOptimizer(exact_dense=True), --exact_adam 1) across the models and
routes: the raw-id catch-up kernel (b2r_adam_exact_catch_up) against the unique-row advance, no new host
synchronisations, NeuMF and SASRec training against dense torch-formula Adam, the evaluation / saving routes, the
single-call BPRMF step and the device-batch epoch."""
import argparse
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu]

DEV = torch.device("cuda", 0)


def _cfg(wd):
    return types.SimpleNamespace(lr=1e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)


def _state(n, d, seed, zero_rows=()):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(n, d, generator=g) * 0.3
    mv = torch.zeros(n, 2, d)
    mv[:, 0] = torch.randn(n, d, generator=g) * 1e-2
    mv[:, 1] = torch.rand(n, d, generator=g) * 1e-4
    mv[list(zero_rows)] = 0.0                               # rows whose moments are zero: only weight decay moves them
    last = torch.randint(0, 30, (n,), generator=g, dtype=torch.int32)
    return W.to(DEV), mv.to(DEV), last.to(DEV)


def _run_catch_up(W, mv, last, ids, upto, stamp, wd, **kw):
    from rechorus_b200 import ops
    W, mv, last = W.clone(), mv.clone(), last.clone()
    d = W.shape[1]
    ops.adam_exact_catch_up(W, mv[:, 0], mv[:, 1], last, ids, upto, _cfg(wd), stamp=stamp, state_ld=2 * d, **kw)
    return W, mv, last


def _run_advance(W, mv, last, rows, upto, stamp, wd):
    from rechorus_b200 import ops
    W, mv, last = W.clone(), mv.clone(), last.clone()
    d = W.shape[1]
    ops.adam_exact_advance(W, mv[:, 0], mv[:, 1], last, upto, _cfg(wd), rows=rows, stamp=stamp, state_ld=2 * d)
    return W, mv, last


# ---------------------------------------------------------------------------------------------------------------------
# 1. the kernel
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("wd", [0.0, 1e-3])
@pytest.mark.parametrize("d", [32, 64, 128])
def test_catch_up_over_raw_ids_equals_advance_over_unique_rows(d, wd):
    """bit for bit in weights, moments and stamps; repeated ids, an ignore id in a prefix, out-of-range ids counted"""
    from rechorus_b200 import ops
    n = 5000
    W, mv, last = _state(n, d, seed=d, zero_rows=range(0, 40))
    g = torch.Generator().manual_seed(d + 1)
    ids = torch.randint(0, 600, (512, 7), generator=g)        # heavy repetition; rows 0..39 have zero moments
    ids[:100, 3] = 7                                          # the ignore id, inside the ignored prefix ...
    ids[400:, 5] = 7                                          # ... and beyond it, where it is an ordinary row
    ids[10, 0], ids[20, 1], ids[30, 2] = -1, n, n + 123        # out of range
    ids = ids.to(DEV)
    ignore_n = 100 * 7
    flat = ids.reshape(-1)
    keep = (flat >= 0) & (flat < n)
    keep[:ignore_n] &= flat[:ignore_n] != 7
    rows = torch.unique(flat[keep])
    flag = ops.err_flag(DEV)
    flag.zero_()
    for stamp in (0, 41):
        a = _run_catch_up(W, mv, last, ids, 40, stamp, wd, ignore_id=7, ignore_n=ignore_n)
        assert int(flag.item()) == 3
        flag.zero_()
        b = _run_advance(W, mv, last, rows, 40, stamp, wd)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        again = _run_catch_up(W, mv, last, ids, 40, stamp, wd, ignore_id=7, ignore_n=ignore_n)
        for x, y in zip(a, again):                            # two runs: identical bits
            assert torch.equal(x, y)
        flag.zero_()
        touched = torch.zeros(n, dtype=torch.bool, device=DEV)
        touched[rows] = True
        assert torch.equal(a[0][~touched], W[~touched]) and torch.equal(a[2][~touched], last[~touched])
        assert bool((a[2][touched] == max(40, stamp)).all())
    moved = (a[0] != W).any(dim=1)
    assert bool(moved[rows[rows >= 40]].any())                # the advance really ran


@pytest.mark.parametrize("d", [32, 64, 128])
def test_catch_up_one_row_taking_a_whole_batch(d):
    """[4096, 100] ids that all name one row: it is advanced exactly once, as the unique-row advance moves it"""
    n = 1000
    W, mv, last = _state(n, d, seed=3 * d)
    last[17] = 2
    ids = torch.full((4096, 100), 17, dtype=torch.int64, device=DEV)
    for wd in (0.0, 1e-3):
        a = _run_catch_up(W, mv, last, ids, 50, 51, wd)
        b = _run_advance(W, mv, last, torch.tensor([17], device=DEV), 50, 51, wd)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        assert int(a[2][17]) == 51 and not torch.equal(a[0][17], W[17])
        again = _run_catch_up(W, mv, last, ids, 50, 51, wd)
        for x, y in zip(a, again):
            assert torch.equal(x, y)


def test_exact_mode_refuses_widths_without_a_catch_up_kernel():
    from rechorus_b200.optim import RowSparseOptimizer
    m = _make("BPRMF", "fused", d=48)
    with pytest.raises(ValueError, match="48 wide"):
        RowSparseOptimizer(m, "Adam", lr=1e-2, exact_dense=True)
    RowSparseOptimizer(m, "Adam", lr=1e-2)                    # the lazy mode keeps its plan route for this width


# ---------------------------------------------------------------------------------------------------------------------
# model builders
# ---------------------------------------------------------------------------------------------------------------------

N_USERS, N_ITEMS, USED_U, USED_I = 200, 300, 150, 200         # ids are drawn below USED_*: the rows above stay untouched
B, C, L = 8, 5, 10


def _make(name, mode, d=64, layers="[64]", scale=30.0, seed=21):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    extra = ["--emb_size", str(d), "--num_neg", str(C - 1), "--table_mode", mode]
    if name == "NeuMF":
        extra += ["--layers", layers]
    if name == "SASRec":
        extra += ["--history_max", str(L), "--num_layers", "2", "--num_heads", "4"]
    a = p.parse_args(extra)
    a.device, a.model_path = DEV, "/tmp/_b2r_exact_models.pt"
    torch.manual_seed(seed)
    m = cls(a, types.SimpleNamespace(n_users=N_USERS, n_items=N_ITEMS)).to(DEV)
    with torch.no_grad():
        for prm in m.parameters():
            prm.mul_(scale)                                   # gradients well above rounding (Adam divides by |g|)
    m.set_table_mode(mode)
    m.train()
    return m


def _feeds(name, n, seed=22):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        f = {"user_id": torch.randint(1, USED_U, (B,), generator=g),
             "item_id": torch.randint(1, USED_I, (B, C), generator=g), "batch_size": B, "phase": "train"}
        if name == "SASRec":
            lengths = torch.randint(1, L + 1, (B,), generator=g)
            width = int(lengths.max())
            hist = torch.randint(1, USED_I, (B, width), generator=g)
            hist[torch.arange(width).view(1, -1) >= lengths.view(-1, 1)] = 0        # right-padded with 0
            f["history_items"], f["lengths"] = hist, lengths
        out.append({k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in f.items()})
    return out


def _contract_step(m, feed):
    m.optimizer.zero_grad()
    loss = m.loss(m(feed))
    loss.backward()
    m.optimizer.step()
    return loss.detach()


# ---------------------------------------------------------------------------------------------------------------------
# 2. no new host synchronisations
# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["BPRMF", "NeuMF", "SASRec"])
def test_exact_step_adds_no_host_synchronisation(name):
    from rechorus_b200.optim import RowSparseOptimizer
    feeds = _feeds(name, 3)

    def raises(exact, route):
        m = _make(name, "fused")
        m.optimizer = RowSparseOptimizer(m, "Adam", lr=1e-2, l2=1e-3, exact_dense=exact)
        step = (lambda f: m.train_step(f)) if route == "train_step" else (lambda f: _contract_step(m, f))
        step(feeds[0])                                        # step 1: the catch-up has something to do from step 2 on
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            loss = step(feeds[1])
            err = None
        except RuntimeError as e:
            err = e
        finally:
            torch.cuda.set_sync_debug_mode(0)
        if err is None:
            assert np.isfinite(float(loss))
        return err

    routes = ["contract"] + (["train_step"] if name == "BPRMF" else [])
    for route in routes:
        lazy = raises(False, route)
        exact = raises(True, route)
        if lazy is None:
            assert exact is None, (route, repr(exact))


# ---------------------------------------------------------------------------------------------------------------------
# 3. NeuMF and SASRec follow dense Adam
# ---------------------------------------------------------------------------------------------------------------------

CASES = [("NeuMF", "[64]"), ("NeuMF", "[64, 32]"), ("SASRec", None)]


@pytest.mark.parametrize("l2", [0.0, 1e-3])
@pytest.mark.parametrize("name,layers", CASES)
def test_exact_mode_follows_dense_adam(name, layers, l2):
    """20 steps with exact_dense=True, flushed, against the same model with dense tables and the optimizer's dense
    torch-formula Adam (b2r_dense_optim) on the same batches; a lazy run is the negative control.  Bars: those of the
    BPRMF exact-mode test (tests/test_gpu_optin_modes.py), 2e-5 with weight decay, without it 2e-4 at most and 2e-6 at
    the 90th percentile.  Adam's eps is 1e-3 here, as in tests/test_gpu_bprmf.py's autograd-route test: the step
    lr * m_hat / (sqrt(v_hat) + eps) is ill-conditioned for gradient entries within a few orders of eps (DESIGN.md §6),
    and the deep models have entries whose gradient is rounding noise -- SASRec's key bias (softmax cancels it exactly),
    the bias of a hidden unit whose ReLU is almost never active.  At eps = 1e-8 Adam turns that noise into steps of lr,
    so two fp32 runs that round differently (a dense against a row-sparse table update) drift apart by far more than
    the bars in those entries (measured on an H100: 0.07 in SASRec's key bias after 20 steps), and through them in the
    tables.  At eps = 1e-3 such noise moves nothing, while the catch-up still has everything to do: a row no batch
    touches decays by ~2e-3 per step under l2 = 1e-3, and a row touched early keeps moving with its momentum.

    SASRec at these weights is more sensitive to rounding still (DESIGN.md §6: deep models are judged against their own
    rounding sensitivity): a 7e-7 difference in the weights changes its batch loss by 2e-5, and Adam carries that into
    ~4e-5 of weight per step.  Traced step by step on an H100, the two runs' largest difference grows from 1e-7 to
    3.8e-4 (l2 = 1e-3) and 1.1e-4 (l2 = 0) over the 20 steps, in the rows and parameters the batches train, while the
    rows only the catch-up moves (never-touched rows, item row 0) stay within 4e-7.  So SASRec's parameters are held to
    1e-3, and the never-touched rows and row 0 of every model to the BPRMF bars."""
    from rechorus_b200.optim import RowSparseOptimizer
    kw = {"layers": layers} if layers else {}
    ex, lz, ctl = _make(name, "fused", **kw), _make(name, "fused", **kw), _make(name, "dense", **kw)
    ex.optimizer = RowSparseOptimizer(ex, "Adam", lr=1e-2, l2=l2, eps=1e-3, exact_dense=True)
    lz.optimizer = RowSparseOptimizer(lz, "Adam", lr=1e-2, l2=l2, eps=1e-3)
    ctl.optimizer = RowSparseOptimizer(ctl, "Adam", lr=1e-2, l2=l2, eps=1e-3)
    feeds = _feeds(name, 20)
    for step, f in enumerate(feeds):
        le, ll, lc = _contract_step(ex, f), _contract_step(lz, f), _contract_step(ctl, f)
        if step == 0:
            assert float(le) == float(lc) == float(ll)
    ex.optimizer.flush()
    ref = dict(ctl.named_parameters())

    def bar_ok(err, loose=(name == "SASRec")):
        if loose:
            return float(err.max()) <= 1e-3
        if l2 > 0:
            return float(err.max()) <= 2e-5
        return float(err.max()) <= 2e-4 and float(err.reshape(-1).quantile(0.9)) <= 2e-6

    for k, v in ex.named_parameters():
        err = (v - ref[k]).abs().detach().float().cpu()
        assert bar_ok(err), (k, float(err.max()))
    # by name: rows no batch ever touched, and SASRec's item row 0 (padding: read, never updated by the plan)
    tables = {"NeuMF": [("mf_u_embeddings.weight", USED_U), ("mf_i_embeddings.weight", USED_I),
                        ("mlp_u_embeddings.weight", USED_U), ("mlp_i_embeddings.weight", USED_I)],
              "SASRec": [("i_embeddings.weight", USED_I)]}[name]
    lazy = dict(lz.named_parameters())
    for k, used in tables:
        rows = [0] + list(range(used, ref[k].shape[0]))
        err = (dict(ex.named_parameters())[k][rows] - ref[k][rows]).abs().detach().cpu()
        assert bar_ok(err, loose=False), (k, float(err.max()))
        miss = (lazy[k][rows] - ref[k][rows]).abs().detach().cpu()
        if l2 > 0:
            # dense Adam decays them; the lazy rule leaves them where they started
            assert float(miss.max()) >= 100 * 2e-5, (k, float(miss.max()))
        else:
            # nothing moves them without weight decay, under any rule
            assert float(miss.max()) == 0.0 and float(err.max()) == 0.0, k
    # rows touched by an early batch only: dense Adam's momentum keeps moving them, the lazy rule does not
    late = torch.zeros(N_ITEMS, dtype=torch.bool, device=DEV)
    for f in feeds[-5:]:
        late[f["item_id"].reshape(-1)] = True
        if name == "SASRec":
            late[f["history_items"].reshape(-1)] = True
    early = torch.zeros(N_ITEMS, dtype=torch.bool, device=DEV)
    early[feeds[0]["item_id"].reshape(-1)] = True
    rows = early & ~late
    assert bool(rows.any())
    k = tables[1][0] if name == "NeuMF" else tables[0][0]
    miss = (lazy[k][rows] - ref[k][rows]).abs().detach().cpu()
    err = (dict(ex.named_parameters())[k][rows] - ref[k][rows]).abs().detach().cpu()
    far = 10 * 1e-3 if name == "SASRec" else 100 * 2e-5
    assert float(miss.max()) >= far and bar_ok(err), (float(miss.max()), float(err.max()))


# ---------------------------------------------------------------------------------------------------------------------
# 4. evaluation and saving see caught-up rows
# ---------------------------------------------------------------------------------------------------------------------

FIT = {"BPRMF": ["--emb_size", "64", "--num_neg", "3"],
       "NeuMF": ["--emb_size", "32", "--layers", "[32, 16]", "--num_neg", "2"],
       "SASRec": ["--emb_size", "32", "--num_layers", "2", "--num_heads", "2", "--history_max", "8", "--num_neg", "2"]}


def _fit_corpus():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import fit_corpus
    return fit_corpus.build()


def _trained(name, tmp_path, exact=True, extra=()):
    """(runner, model, corpus, args): one runner epoch in exact mode, not flushed"""
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(FIT[name] + ["--batch_size", "64", "--eval_batch_size", "32", "--num_workers", "0", "--lr", "0.01",
                                  "--l2", "1e-3", "--fused_optimizer", "1", "--exact_adam", str(int(exact)), "--topk",
                                  "5,10", "--metric", "NDCG,HR", "--epoch", "1", *extra])
    a.device, a.model_path, a.log_file = DEV, str(tmp_path / f"{name}_{len(os.listdir(tmp_path))}.pt"), ""
    corpus = _fit_corpus()
    np.random.seed(5)
    torch.manual_seed(5)
    model = cls(a, corpus).to(DEV)
    runner = BaseRunner(a)
    train = cls.Dataset(model, corpus, "train")
    runner.fit(train, epoch=1)
    return runner, model, corpus, a


def _flushed_reference(name, tmp_path):
    """a plain dense-table model holding the flushed weights of the same training"""
    from rechorus_b200 import plugin
    runner, model, corpus, a = _trained(name, tmp_path)
    raw = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model.optimizer.flush()
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert any(not torch.equal(raw[k], sd[k]) for k in sd)    # the flush moves rows: the checks below have teeth
    a.exact_adam, a.fused_optimizer = 0, 0
    ref = getattr(plugin, name)(a, corpus).to(DEV)
    ref.load_state_dict(sd)
    ref.eval()
    return runner, ref, corpus, sd


def _eval_set(model, corpus):
    ds = type(model).Dataset(model, corpus, "dev")
    ds.prepare()
    return ds


@pytest.mark.parametrize("name", ["BPRMF", "NeuMF", "SASRec"])
def test_evaluation_and_saving_see_caught_up_rows(name, tmp_path):
    from rechorus_b200.runner import device_eval_batches
    runner, ref, corpus, sd = _flushed_reference(name, tmp_path)
    want_pred = runner.predict(_eval_set(ref, corpus))
    ref_ds = _eval_set(ref, corpus)
    want_ranks = torch.cat([ref.eval_ranks(f, clicked=c).clone() for f, c in device_eval_batches(ref_ds, 32)])
    want_rec = runner.recommend(_eval_set(ref, corpus), 5)

    # the host predict route: forward in eval mode through ``inference``
    r, m, _, _ = _trained(name, tmp_path)
    assert np.array_equal(r.predict(_eval_set(m, corpus)), want_pred)
    # --device_metrics 1 ranks
    r, m, _, _ = _trained(name, tmp_path)
    m.eval()
    got = torch.cat([m.eval_ranks(f, clicked=c).clone() for f, c in device_eval_batches(_eval_set(m, corpus), 32)])
    assert torch.equal(got, want_ranks)
    # recommend lists
    r, m, _, _ = _trained(name, tmp_path)
    got = r.recommend(_eval_set(m, corpus), 5)
    assert got[0] == want_rec[0] and np.array_equal(got[1], want_rec[1]) and np.array_equal(got[2], want_rec[2])
    # the checkpoint save_model writes (here straight after training, in train mode)
    r, m, _, a = _trained(name, tmp_path)
    m.save_model()
    ck = torch.load(a.model_path, map_location=DEV)
    for k, v in sd.items():
        assert torch.equal(ck[k], v), k


@pytest.mark.parametrize("name", ["BPRMF", "SASRec"])
def test_runner_train_loop_checkpoint_holds_flushed_weights(name, tmp_path):
    """BaseRunner.train: fit, evaluate, save_model -- the saved checkpoint is the flushed model"""
    _, _, corpus, sd = _flushed_reference(name, tmp_path)
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = getattr(plugin, name)
    p = cls.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
    a = p.parse_args(FIT[name] + ["--batch_size", "64", "--eval_batch_size", "32", "--num_workers", "0", "--lr", "0.01",
                                  "--l2", "1e-3", "--fused_optimizer", "1", "--exact_adam", "1", "--topk", "5,10",
                                  "--metric", "NDCG,HR", "--epoch", "1"])
    a.device, a.model_path, a.log_file = DEV, str(tmp_path / "train_loop.pt"), ""
    np.random.seed(5)
    torch.manual_seed(5)
    model = cls(a, corpus).to(DEV)
    runner = BaseRunner(a)
    data = {ph: cls.Dataset(model, corpus, ph) for ph in ("train", "dev", "test")}
    data["dev"].prepare()
    data["test"].prepare()
    runner.train(data)
    ck = torch.load(a.model_path, map_location=DEV)
    for k, v in sd.items():
        assert torch.equal(ck[k], v), k


# ---------------------------------------------------------------------------------------------------------------------
# 5. the single-call BPRMF step
# ---------------------------------------------------------------------------------------------------------------------

def test_single_call_step_runs_exact_mode_and_matches_the_autograd_route():
    """--fused_step 1 --exact_adam 1: b2r_bprmf_train_step at config 2's shape (1M x 1M rows, d = 64, B = 4096, C = 100)
    with l2 > 0, never the autograd fallback; same tables as forward -> backward -> RowSparseOptimizer.step() in exact
    mode, within the bars of the lazy whole-step-versus-contract-route test (tests/test_gpu_c2_step.py)"""
    from rechorus_b200 import plugin
    from rechorus_b200.optim import RowSparseOptimizer
    from rechorus_b200.runner import BaseRunner
    nu = ni = 1_000_000
    Bc, Cc = 4096, 100

    def model():
        p = plugin.BPRMF.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
        a = p.parse_args(["--emb_size", "64", "--num_neg", str(Cc - 1), "--table_mode", "fused"])
        a.device, a.model_path = DEV, "/tmp/_b2r_unused.pt"
        torch.manual_seed(0)
        m = plugin.BPRMF(a, types.SimpleNamespace(n_users=nu, n_items=ni)).to(DEV)
        with torch.no_grad():
            for q in m.parameters():
                q.mul_(20.0)
        m.optimizer = RowSparseOptimizer(m, "Adam", lr=1e-3, l2=1e-4, exact_dense=True)
        m.train()
        return m

    g = torch.Generator().manual_seed(31)
    feeds = []
    for _ in range(4):
        uid = torch.randint(1, nu, (Bc,), generator=g)
        iid = torch.randint(1, ni, (Bc, Cc), generator=g)
        uid[: Bc // 2] = uid[: Bc // 2] % 5000 + 1            # rows shared between steps: their catch-up matters
        iid[:, :10] = iid[:, :10] % 20000 + 1
        feeds.append({"user_id": uid.to(DEV), "item_id": iid.to(DEV), "batch_size": Bc, "phase": "train"})
    ma, mb = model(), model()

    def no_fallback(*a, **k):
        raise AssertionError("train_step fell back to the autograd route")

    mb.forward = no_fallback
    for t, f in enumerate(feeds):
        la = _contract_step(ma, f)
        lb = mb.train_step(f, feeds[t + 1] if t + 1 < len(feeds) else None)
        assert abs(float(la) - float(lb)) <= 2e-6, t
    for mm in (ma, mb):
        assert mm.optimizer.t == len(feeds)
    ea, eb = ma.optimizer.entry(ma.i_embeddings.weight), mb.optimizer.entry(mb.i_embeddings.weight)
    assert torch.equal(ea["last"], eb["last"])
    ma.optimizer.flush()
    mb.optimizer.flush()
    for (k, pa), (_, pb) in zip(ma.named_parameters(), mb.named_parameters()):
        assert (pa - pb).abs().max() <= 1e-6, k


# ---------------------------------------------------------------------------------------------------------------------
# 6. device-built batches
# ---------------------------------------------------------------------------------------------------------------------

def test_sasrec_exact_device_epoch_equals_the_same_batches_fed_by_hand():
    from rechorus_b200 import ops, plugin
    from rechorus_b200.optim import RowSparseOptimizer
    from rechorus_b200.runner import BaseRunner
    flags = FIT["SASRec"] + ["--batch_size", "64", "--num_workers", "0", "--lr", "0.01", "--l2", "1e-3",
                             "--table_mode", "fused", "--fused_optimizer", "1", "--exact_adam", "1",
                             "--device_batches", "77"]
    corpus = _fit_corpus()

    def build():
        p = plugin.SASRec.parse_model_args(BaseRunner.parse_runner_args(argparse.ArgumentParser()))
        a = p.parse_args(flags)
        a.device, a.model_path, a.log_file = DEV, "/tmp/_b2r_exact_db.pt", ""
        torch.manual_seed(1)
        model = plugin.SASRec(a, corpus).to(DEV)
        return model, plugin.SASRec.Dataset(model, corpus, "train"), BaseRunner(a)

    model, train, runner = build()
    l1 = runner.fit(train, epoch=1)
    assert model.optimizer.exact_dense
    st = train.__dict__["_b2r_dev"]
    N, K, Bn, Lp = st["users"].numel(), 2, 64, st["history"].width
    neg = st["sampler"].sample(st["users"], K, 1)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(st["seed"] * 1_000_003 + 1)
    perm = torch.randperm(N, device="cuda", generator=gen)
    model2, train2, _ = build()
    train2.data["neg_items"] = neg.cpu().numpy()
    model2.optimizer = RowSparseOptimizer(model2, "Adam", lr=0.01, l2=1e-3, exact_dense=True)
    model2.set_table_mode("fused")
    model2.train()
    losses = []
    for k in range((N + Bn - 1) // Bn):
        rows = perm[k * Bn:(k + 1) * Bn]
        host = train2.collate_batch([train2._get_feed_dict(int(r)) for r in rows.tolist()])
        feed = {"user_id": host["user_id"].cuda(), "item_id": host["item_id"].cuda(), "lengths": host["lengths"].cuda(),
                "history_items": F.pad(host["history_items"], (0, Lp - host["history_items"].shape[1])).cuda(),
                "batch_size": rows.numel(), "phase": "train"}
        losses.append(_contract_step(model2, feed))
    assert abs(float(torch.stack(losses).mean()) - l1) <= 1e-6
    for (k, pa), (_, pb) in zip(model.named_parameters(), model2.named_parameters()):
        assert torch.equal(pa, pb), k
    model.optimizer.flush()
    model2.optimizer.flush()
    for (k, pa), (_, pb) in zip(model.named_parameters(), model2.named_parameters()):
        assert torch.equal(pa, pb), k
    ops.check_ids()
