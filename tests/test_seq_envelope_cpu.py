"""CPU: SASRec's training envelope.  b2r_seq_train_check answers from the launchers' own shape predicates, and a SASRec
whose training step some kernel would refuse is refused at construction (ValueError), not by its first backward."""
import argparse
import types

import pytest
import torch

LASTQ, V1 = 1, 2                     # B2R_SEQ_LAST_QUERY, B2R_SEQ_ATTN_V1


@pytest.fixture(scope="module")
def lib():
    from rechorus_b200 import build
    from rechorus_b200 import lib as L
    build.build()
    return L.load()


# (L, d, H, full_blocks, flags) -> (return code, kernel named in the message)
QUERY_CASES = [
    # register-resident backward: (5 L (d + 4) + 2 L H) * 4 B <= 227 KB
    ((86, 128, 4, 1, 0), 0, None),
    ((87, 128, 4, 1, 0), -3, "b2r_attention_bwd_rt"),
    ((85, 128, 8, 1, 0), 0, None),
    ((86, 128, 8, 1, 0), -3, "b2r_attention_bwd_rt"),
    ((114, 96, 3, 1, 0), 0, None),
    ((115, 96, 3, 1, 0), -3, "b2r_attention_bwd_rt"),
    ((128, 96, 3, 1, 0), -3, "b2r_attention_bwd_rt"),
    ((44, 256, 8, 1, 0), 0, None),
    ((50, 256, 8, 1, 0), -3, "b2r_attention_bwd_rt"),
    # full attention needs L <= 128 on either route
    ((128, 64, 4, 1, 0), 0, None),
    ((129, 64, 4, 1, 0), -3, "b2r_attention_bwd_live"),
    ((128, 32, 1, 1, 0), 0, None),
    # d / H = 64 always takes the shared-memory kernels: (4 L (d + 1) + H L (L + 1)) * 4 B <= 227 KB
    ((128, 64, 1, 1, 0), 0, None),
    ((84, 128, 2, 1, 0), 0, None),
    ((85, 128, 2, 1, 0), -3, "b2r_attention_bwd_live"),
    ((47, 256, 4, 1, 0), 0, None),
    ((48, 256, 4, 1, 0), -3, "b2r_attention_bwd_live"),
    # the shared-memory kernels forced for every shape
    ((128, 64, 4, 1, V1), -3, "b2r_attention_bwd_live"),
    ((128, 32, 1, 1, V1), 0, None),
    # one 1-block SASRec: last-query block only, the position table has no limit of its own
    ((200, 64, 4, 0, LASTQ), 0, None),
    ((256, 64, 4, 0, LASTQ), 0, None),
    ((256, 256, 8, 0, LASTQ), 0, None),
    ((257, 64, 4, 0, LASTQ), -3, "b2r_attention_last"),
    # residual LayerNorm backward: d <= 256
    ((50, 288, 4, 0, LASTQ), -3, "b2r_add_layernorm_bwd"),
    ((50, 288, 4, 1, 0), -3, "b2r_add_layernorm_bwd"),
    # bad arguments
    ((0, 64, 4, 1, 0), -1, "b2r_seq_train_check"),
    ((50, 64, 3, 1, 0), -1, "b2r_seq_train_check"),
    ((50, 64, 4, -1, 0), -1, "b2r_seq_train_check"),
    ((50, 64, 4, 1, 4), -1, "b2r_seq_train_check"),
]


@pytest.mark.parametrize("args,rc,kernel", QUERY_CASES)
def test_seq_train_check_answers_the_boundary_cases(lib, args, rc, kernel):
    assert lib.b2r_seq_train_check(*args) == rc
    if kernel is not None:
        assert kernel in lib.b2r_last_error().decode()


def test_seq_train_check_is_monotone_in_the_batch_width(lib):
    """a batch is padded to its longest history, so accepting L must accept every narrower width"""
    for d, H in ((32, 4), (64, 4), (64, 1), (96, 3), (128, 4), (128, 8), (128, 2), (256, 8)):
        ok = [lib.b2r_seq_train_check(L, d, H, 1, 0) == 0 for L in range(1, 140)]
        first_bad = ok.index(False) if False in ok else len(ok)
        assert all(ok[:first_bad]) and not any(ok[first_bad:]), (d, H)


def _build(d, H, layers, hm):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    p = plugin.SASRec.parse_model_args(p)
    a = p.parse_args(["--emb_size", str(d), "--num_heads", str(H), "--num_layers", str(layers),
                      "--history_max", str(hm)])
    a.device, a.model_path = torch.device("cpu"), "/tmp/_b2r_unused.pt"
    return plugin.SASRec(a, types.SimpleNamespace(n_users=10, n_items=300))


# the model-level grid of tests/test_gpu_seq_envelope.py: (emb_size, num_heads, num_layers, history_max, last_query)
ACCEPTED = [(64, 4, 2, 128, True), (64, 4, 2, 128, False), (64, 4, 1, 200, True), (64, 4, 1, 256, True),
            (128, 4, 2, 86, True), (128, 4, 2, 86, False), (64, 1, 2, 100, True), (64, 1, 2, 100, False),
            (32, 1, 2, 128, True), (32, 1, 2, 128, False), (128, 2, 2, 64, True), (128, 2, 2, 64, False),
            (256, 8, 1, 50, True), (64, 4, 2, 50, True), (64, 4, 2, 50, False)]
REFUSED = [(64, 4, 2, 129, True), (128, 4, 2, 87, True), (64, 4, 1, 257, True), (256, 8, 2, 50, True),
           (64, 4, 1, 200, False), (64, 4, 1, 256, False), (256, 8, 1, 50, False), (128, 4, 1, 87, False),
           (288, 4, 1, 20, True)]


@pytest.mark.parametrize("d,H,layers,hm,lastq", ACCEPTED)
def test_sasrec_in_the_envelope_constructs(monkeypatch, lib, d, H, layers, hm, lastq):
    from rechorus_b200 import plugin
    monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
    m = _build(d, H, layers, hm)
    assert m.p_embeddings.weight.shape == (hm + 1, d)


@pytest.mark.parametrize("d,H,layers,hm,lastq", REFUSED)
def test_sasrec_outside_the_envelope_is_refused_at_construction(monkeypatch, lib, d, H, layers, hm, lastq):
    from rechorus_b200 import plugin
    monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
    with pytest.raises(ValueError) as e:
        _build(d, H, layers, hm)
    msg = str(e.value)
    assert f"history_max={hm}" in msg and f"emb_size={d}" in msg and f"num_heads={H}" in msg
    assert "b2r_" in msg                                     # the library's reason: which kernel, which limit


def test_forcing_the_shared_memory_attention_kernels_narrows_the_envelope(monkeypatch, lib):
    from rechorus_b200 import ops, plugin
    monkeypatch.setattr(plugin, "_SASREC_LASTQ", True)
    _build(64, 4, 2, 128)
    monkeypatch.setattr(ops, "_ATTN_RT", False)
    with pytest.raises(ValueError, match="b2r_attention_bwd_live"):
        _build(64, 4, 2, 128)
