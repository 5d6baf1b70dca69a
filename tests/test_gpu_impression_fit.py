"""GPU: impression training on device-built batches -- b2r_collate_impression_train against the batches the reference's
ImpressionRunner.fit passes its model (fixture), its null-permutation path against b2r_collate_impression, argument
checks, and runner.fit_impression_on_device for BPRMFImpression and SASRecImpression against a host route (the real
DataLoader over the oracle's collate and labels): identical epoch losses, parameters and CPU RNG state."""
import argparse
import types

import numpy as np
import pytest
import torch

from tests.impression_oracle import impression_collate, impression_history
from tests.test_impression_fit_cpu import GOLDEN, TAGS, fixture_rows, impression_labels

pytestmark = [pytest.mark.gpu]
DEV = torch.device("cuda", 0)


class _Recorder:
    """a kernel-free model for fit_impression_on_device: records every batch and label tensor it is given"""

    def __init__(self, mp, mn, H=None):
        self.device, self.train_max_pos_item, self.train_max_neg_item = DEV, mp, mn
        if H is not None:
            self.history_max = H
        self.optimizer = types.SimpleNamespace(zero_grad=lambda: None, step=lambda: None)
        self.batches = []

    def train(self, mode=True):
        return self

    def __call__(self, feed):
        self.batches.append({k: v.cpu().numpy() for k, v in feed.items() if isinstance(v, torch.Tensor)})
        return {"prediction": torch.zeros(feed["item_id"].shape, device=DEV)}

    def loss(self, out, target):
        self.batches[-1]["labels"] = target.cpu().numpy()
        return torch.zeros((), device=DEV, requires_grad=True)


def _dataset(model, users, position, pos, neg, his, n_users):
    data = {"user_id": [int(u) for u in users], "pos_items": pos, "neg_items": neg,
            "position": [int(p) for p in position], "pos_num": [len(x) for x in pos], "neg_num": [len(x) for x in neg]}
    corpus = types.SimpleNamespace(user_his={u: {"pos": h, "neg": []} for u, h in his.items()}, n_users=n_users)
    return types.SimpleNamespace(model=model, corpus=corpus, data=data, phase="train", actions_before_epoch=lambda: None)


@pytest.mark.parametrize("tag", TAGS)
def test_device_epochs_equal_the_reference_fit_batches(tag):
    from rechorus_b200 import ops
    from rechorus_b200.runner import fit_impression_on_device
    z = np.load(GOLDEN)
    mp, mn, B, H = (int(z[k]) for k in ("mp", "mn", "B", "history_max"))
    _, users, position, pos, neg, his = fixture_rows(z, tag)
    model = _Recorder(mp, mn, H if tag == "seq" else None)
    ds = _dataset(model, users, position, pos, neg, his, int(z["n_users"]))
    runner = types.SimpleNamespace(batch_size=B)
    torch.manual_seed(int(z["seed"]))
    for e in range(1, int(z["epochs"]) + 1):
        model.batches = []
        assert fit_impression_on_device(runner, ds, e) == 0.0
        assert len(model.batches) == (len(users) + B - 1) // B
        for bi, b in enumerate(model.batches):
            keys = ("user_id", "item_id", "labels") + (("history_items", "lengths") if tag == "seq" else ())
            for k in keys:
                assert b[k].dtype == np.int64 and np.array_equal(b[k], z[f"{tag}/{e}/{bi}/{k}"]), (e, bi, k)
        assert np.array_equal(torch.get_rng_state().numpy(), z[f"{tag}/{e}/rng"]), e
    ops.check_ids()


def _device_csr(rng, N, mp, mn, n_users):
    from rechorus_b200 import ops
    pos = [list(rng.randint(1, 1000, rng.randint(0, mp + 4))) for _ in range(N)]
    neg = [list(rng.randint(1, 1000, rng.randint(0, mn + 4))) for _ in range(N)]
    up = lambda a: torch.as_tensor(np.asarray(a, dtype=np.int64)).to(DEV)      # noqa: E731
    pp, pi = ops.list_csr(pos, mp)
    npt, ni = ops.list_csr(neg, mn)
    pn = rng.randint(0, mp + 4, N)
    nn = rng.randint(0, mn + 4, N)
    return pos, neg, pn, nn, (up(rng.randint(0, n_users, N)), up(pp), up(pi), up(npt), up(ni), up(pn), up(nn))


@pytest.mark.parametrize("mp,mn", [(1, 1), (3, 7), (20, 20), (20, 0), (0, 5)])
def test_null_permutation_equals_collate_impression_and_labels_restate_fit(mp, mn):
    from rechorus_b200 import ops
    rng = np.random.RandomState(mp * 100 + mn)
    N, n_users, B = 301, 40, 64
    pos, neg, pn, nn, (users, pp, pi, npt, ni, pnd, nnd) = _device_csr(rng, N, mp, mn, n_users)
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(mp + mn)).to(DEV)
    for start in range(0, N, B):
        Bn = min(B, N - start)
        u1, i1 = torch.empty(B, dtype=torch.int64, device=DEV), torch.empty((B, mp + mn), dtype=torch.int64, device=DEV)
        u2, i2, l2 = torch.empty_like(u1), torch.empty_like(i1), torch.empty_like(i1)
        ops.collate_impression(users, pp, pi, npt, ni, n_users, start, Bn, mp, mn, u1, i1)
        ops.collate_impression_train(users, pp, pi, npt, ni, pnd, nnd, None, n_users, start, Bn, mp, mn, u2, i2, l2)
        assert torch.equal(u1[:Bn], u2[:Bn]) and torch.equal(i1[:Bn], i2[:Bn])
        r = np.arange(start, start + Bn)
        assert np.array_equal(l2[:Bn].cpu().numpy(), impression_labels(pn[r], nn[r], mp, mn))
        # a permutation: the same rows, gathered
        ops.collate_impression_train(users, pp, pi, npt, ni, pnd, nnd, perm, n_users, start, Bn, mp, mn, u2, i2, l2)
        r = perm[start:start + Bn].cpu().numpy()
        uid, iid = impression_collate([pos[i] for i in r], [neg[i] for i in r], users.cpu().numpy()[r], mp, mn)
        assert np.array_equal(u2[:Bn].cpu().numpy(), uid) and np.array_equal(i2[:Bn].cpu().numpy(), iid)
        assert np.array_equal(l2[:Bn].cpu().numpy(), impression_labels(pn[r], nn[r], mp, mn))
    ops.check_ids()


def test_bad_arguments_are_rejected_and_bad_users_raise_at_the_poll():
    from rechorus_b200 import lib, ops
    rng = np.random.RandomState(1)
    N, mp, mn = 10, 2, 3
    _, _, _, _, (users, pp, pi, npt, ni, pn, nn) = _device_csr(rng, N, mp, mn, 5)
    perm = torch.arange(N, device=DEV)
    u, i = torch.empty(4, dtype=torch.int64, device=DEV), torch.empty((4, mp + mn), dtype=torch.int64, device=DEV)
    lab = torch.empty_like(i)
    args = [users, pp, pi, npt, ni, pn, nn, perm, 5, 0, 4, mp, mn, u, i, lab]

    def call(**kw):
        a = list(args)
        for k, v in kw.items():
            a[int(k[1:])] = v
        ops.collate_impression_train(*a)

    for bad in (dict(a15=torch.empty((4, mp + mn + 1), dtype=torch.int64, device=DEV)),   # labels wider than the batch
                dict(a14=torch.empty((3, mp + mn), dtype=torch.int64, device=DEV)),       # fewer rows than Bn
                dict(a7=perm[:N - 1].contiguous()),                                       # perm shorter than the set
                dict(a5=pn[:N - 1].contiguous()),                                         # pos_num shorter than the set
                dict(a9=8)):                                                              # batch past the last row
        with pytest.raises(ValueError):
            call(**bad)
    with pytest.raises(TypeError):
        call(a15=lab.int())
    L = lib.load()
    assert L.b2r_collate_impression_train(users.data_ptr(), pp.data_ptr(), pi.data_ptr(), npt.data_ptr(), ni.data_ptr(),
                                          None, nn.data_ptr(), None, 5, 0, 4, mp, mn, u.data_ptr(), i.data_ptr(),
                                          lab.data_ptr(), None, None) == -1
    ops.check_ids()
    users[3] = 99
    call()
    with pytest.raises(IndexError):
        ops.check_ids()
    ops.check_ids()


# ---- fit_impression_on_device against the host route ---------------------------------------------------------------

N_USERS, N_ITEMS = 50, 120
MODELS = {"BPRMFImpression": ["--emb_size", "64"],
          "SASRecImpression": ["--emb_size", "64", "--num_layers", "1", "--num_heads", "1", "--history_max", "20"]}


def _impression_data(N, mp, mn, seed):
    rng = np.random.RandomState(seed)
    his = {u: [(int(i), t) for t, i in enumerate(rng.randint(1, N_ITEMS, rng.randint(1, 40)))] for u in range(1, N_USERS)}
    users = rng.randint(1, N_USERS, N)
    pos = [[int(x) for x in rng.randint(1, N_ITEMS, rng.randint(1, mp + 5))] for _ in range(N)]
    neg = [[int(x) for x in rng.randint(1, N_ITEMS, rng.randint(1, mn + 5))] for _ in range(N)]
    position = [int(rng.randint(1, len(his[int(u)]) + 1)) for u in users]
    return users, position, pos, neg, his


def _model(name, mp, mn, loss_n, dropout):
    from rechorus_b200 import plugin
    cls = getattr(plugin, name)
    flags = [*MODELS[name], "--train_max_pos_item", str(mp), "--train_max_neg_item", str(mn), "--loss_n", loss_n]
    if dropout:
        flags += ["--dropout", str(dropout)]
    a = cls.parse_model_args(argparse.ArgumentParser()).parse_args(flags)
    a.device, a.model_path = DEV, "/tmp/_b2r_imp_fit.pt"
    torch.manual_seed(3)
    return cls(a, types.SimpleNamespace(n_users=N_USERS, n_items=N_ITEMS)).to(DEV)


def _build_optimizer(model):
    return torch.optim.Adam(model.customize_parameters(), lr=0.01)


def _host_fit(model, ds, B):
    """ImpressionRunner.fit's loop: the real DataLoader shuffle, the oracle's collate and labels, host-to-device copies"""
    from torch.utils.data import DataLoader
    d = ds.data
    if model.optimizer is None:
        model.optimizer = _build_optimizer(model)
    model.train()
    mp, mn = model.train_max_pos_item, model.train_max_neg_item
    losses = []
    for r in DataLoader(list(range(len(d["user_id"]))), batch_size=B, shuffle=True, num_workers=0, collate_fn=list):
        uid, iid = impression_collate([d["pos_items"][i] for i in r], [d["neg_items"][i] for i in r],
                                      [d["user_id"][i] for i in r], mp, mn)
        lab = impression_labels([d["pos_num"][i] for i in r], [d["neg_num"][i] for i in r], mp, mn)
        feed = {"user_id": torch.from_numpy(uid).to(DEV), "item_id": torch.from_numpy(iid).to(DEV),
                "batch_size": len(r), "phase": "train"}
        if hasattr(model, "history_max"):
            his = {u: h["pos"] for u, h in ds.corpus.user_his.items()}
            hi, ln = impression_history(his, uid, [d["position"][i] for i in r], model.history_max)
            feed["history_items"], feed["lengths"] = torch.from_numpy(hi).to(DEV), torch.from_numpy(ln).to(DEV)
        model.optimizer.zero_grad()
        out = model(feed)
        loss = model.loss(out, torch.from_numpy(lab).to(DEV))
        loss.backward()
        model.optimizer.step()
        losses.append(loss.detach().cpu().data.numpy())
    return np.mean(losses).item()


CASES = [("BPRMFImpression", "BPR", 0), ("BPRMFImpression", "softmaxCE", 0), ("SASRecImpression", "BPR", 0),
         ("SASRecImpression", "softmaxCE", 0), ("SASRecImpression", "BPR", 0.2), ("SASRecImpression", "softmaxCE", 0.2)]


@pytest.mark.parametrize("name,loss_n,dropout", CASES)
def test_fit_on_device_equals_host_route(name, loss_n, dropout):
    from rechorus_b200.runner import fit_impression_on_device
    mp, mn, N, B = 5, 7, 517, 64
    users, position, pos, neg, his = _impression_data(N, mp, mn, seed=len(name) + len(loss_n))
    dev_model, host_model = _model(name, mp, mn, loss_n, dropout), _model(name, mp, mn, loss_n, dropout)
    ds_dev = _dataset(dev_model, users, position, pos, neg, his, N_USERS)
    ds_host = _dataset(host_model, users, position, pos, neg, his, N_USERS)
    runner = types.SimpleNamespace(batch_size=B, _build_optimizer=_build_optimizer)
    torch.manual_seed(11)
    dev_losses = [fit_impression_on_device(runner, ds_dev, e) for e in (1, 2)]
    dev_rng = torch.get_rng_state()
    torch.manual_seed(11)
    host_losses = [_host_fit(host_model, ds_host, B) for _ in (1, 2)]
    assert dev_losses == host_losses and all(np.isfinite(dev_losses)) and dev_losses[0] != dev_losses[1]
    assert torch.equal(dev_rng, torch.get_rng_state())
    for (k, a), (_, b) in zip(dev_model.named_parameters(), host_model.named_parameters()):
        assert torch.equal(a, b), k


class _NaNOnce(_Recorder):
    """a NaN prediction in the second step"""

    def __call__(self, feed):
        out = super().__call__(feed)
        if len(self.batches) == 2:
            out["prediction"][0, 0] = float("nan")
        return out


def test_non_finite_steps_are_logged_and_training_goes_on(caplog):
    import logging

    from rechorus_b200.runner import fit_impression_on_device
    mp, mn, N, B = 2, 2, 10, 4
    users, position, pos, neg, his = _impression_data(N, mp, mn, seed=4)
    model = _NaNOnce(mp, mn)
    ds = _dataset(model, users, position, pos, neg, his, N_USERS)
    with caplog.at_level(logging.INFO):
        loss = fit_impression_on_device(types.SimpleNamespace(batch_size=B), ds, 6)
    assert loss == 0.0 and len(model.batches) == 3
    assert [r.getMessage() for r in caplog.records if "Nan" in r.getMessage()] == ["Loss is Nan. Stop training at 7."]


def test_a_200k_row_epoch_completes():
    from rechorus_b200 import ops
    from rechorus_b200.runner import fit_impression_on_device
    mp = mn = 20
    N, B = 200_000, 256
    rng = np.random.RandomState(0)
    users = rng.randint(1, N_USERS, N)
    pos = [list(x) for x in np.split(rng.randint(1, N_ITEMS, 25 * N), N)]
    neg = [list(x) for x in np.split(rng.randint(1, N_ITEMS, 25 * N), N)]
    model = _model("BPRMFImpression", mp, mn, "BPR", 0)
    ds = _dataset(model, users, [1] * N, pos, neg, {}, N_USERS)
    loss = fit_impression_on_device(types.SimpleNamespace(batch_size=B, _build_optimizer=_build_optimizer), ds, 1)
    assert np.isfinite(loss)
    ops.check_ids()
