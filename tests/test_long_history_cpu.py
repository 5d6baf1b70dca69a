"""CPU: SASRec's envelope with --tiled_attention.  b2r_seq_train_check_tiled admits every shape b2r_seq_train_check
admits and, beyond it, the widths the tiled attention kernels take; a SASRec outside the default envelope but inside the
tiled one constructs with the flag, is refused without it, and the refusal names the flag."""
import argparse
import types

import pytest
import torch

from tests.test_seq_envelope_cpu import REFUSED

LASTQ = 1                            # B2R_SEQ_LAST_QUERY


@pytest.fixture(scope="module")
def lib():
    from rechorus_b200 import build
    from rechorus_b200 import lib as L
    build.build()
    return L.load()


# (L, d, H, full_blocks, flags) -> (return code, kernel or limit named in the message)
TILED_CASES = [
    ((129, 64, 4, 1, 0), 0, None),
    ((87, 128, 4, 1, 0), 0, None),
    ((257, 64, 4, 0, LASTQ), 0, None),
    ((1024, 64, 1, 2, LASTQ), 0, None),
    ((300, 256, 8, 1, 0), 0, None),
    ((65535, 64, 4, 1, 0), 0, None),
    ((65535, 64, 4, 0, LASTQ), 0, None),
    ((200, 64, 2, 1, 0), 0, None),
    ((128, 96, 3, 1, 0), 0, None),
    # refusals
    ((300, 288, 4, 1, 0), -3, "b2r_add_layernorm_bwd"),
    ((50, 288, 4, 0, LASTQ), -3, "b2r_add_layernorm_bwd"),
    ((65536, 64, 4, 1, 0), -3, "b2r_dropout"),
    ((65536, 64, 4, 0, LASTQ), -3, "b2r_dropout"),
    ((129, 96, 4, 1, 0), -3, "b2r_attention_fwd_tiled"),
    ((129, 24, 1, 1, 0), -3, "b2r_attention_fwd_tiled"),
    ((200, 128, 1, 1, 0), -3, "b2r_attention_fwd_tiled"),
    # no attention block: no width limit, as in the default check
    ((70000, 64, 4, 0, 0), 0, None),
    # bad arguments
    ((0, 64, 4, 1, 0), -1, "b2r_seq_train_check_tiled"),
    ((50, 64, 3, 1, 0), -1, "b2r_seq_train_check_tiled"),
    ((50, 62, 2, 1, 0), -1, "b2r_seq_train_check_tiled"),
    ((50, 64, 4, -1, 0), -1, "b2r_seq_train_check_tiled"),
    ((50, 64, 4, 1, 2), -1, "b2r_seq_train_check_tiled"),
]


@pytest.mark.parametrize("args,rc,kernel", TILED_CASES)
def test_seq_train_check_tiled_answers_the_boundary_cases(lib, args, rc, kernel):
    assert lib.b2r_seq_train_check_tiled(*args) == rc
    if kernel is not None:
        assert kernel in lib.b2r_last_error().decode()


GRID_DH = [(32, 4), (32, 1), (64, 4), (64, 1), (64, 2), (96, 3), (96, 4), (128, 4), (128, 8), (128, 2), (128, 1),
           (256, 8), (256, 4), (256, 32), (288, 9)]


def test_seq_train_check_tiled_is_a_superset_of_the_default_check(lib):
    for d, H in GRID_DH:
        for L in list(range(1, 300, 7)) + [256, 257, 512, 1024]:
            for blocks in (0, 1, 3):
                for flags in (0, LASTQ):
                    if lib.b2r_seq_train_check(L, d, H, blocks, flags) == 0:
                        assert lib.b2r_seq_train_check_tiled(L, d, H, blocks, flags) == 0, (L, d, H, blocks, flags)


def test_seq_train_check_tiled_is_monotone_in_the_batch_width(lib):
    """a batch is padded to its longest history, so accepting L must accept every narrower width"""
    for d, H in GRID_DH:
        for blocks, flags in ((1, 0), (1, LASTQ), (0, LASTQ)):
            ok = [lib.b2r_seq_train_check_tiled(L, d, H, blocks, flags) == 0 for L in range(1, 600)]
            first_bad = ok.index(False) if False in ok else len(ok)
            assert all(ok[:first_bad]) and not any(ok[first_bad:]), (d, H, blocks, flags)


def _build(d, H, layers, hm, tiled=None, cls=None):
    from rechorus_b200 import plugin
    from rechorus_b200.runner import BaseRunner
    cls = cls or plugin.SASRec
    p = BaseRunner.parse_runner_args(argparse.ArgumentParser())
    p = cls.parse_model_args(p)
    argv = ["--emb_size", str(d), "--num_heads", str(H), "--num_layers", str(layers), "--history_max", str(hm)]
    if tiled is not None:
        argv += ["--tiled_attention", str(tiled)]
    a = p.parse_args(argv)
    a.device, a.model_path = torch.device("cpu"), "/tmp/_b2r_unused.pt"
    return cls(a, types.SimpleNamespace(n_users=10, n_items=300))


def _tiled_admits(lib, d, H, layers, hm, lastq):
    return lib.b2r_seq_train_check_tiled(hm, d, H, layers - int(lastq), LASTQ if lastq else 0) == 0


ADMITTED = [c for c in REFUSED if c[0] <= 256 and (c[0] // c[1]) in (8, 16, 32, 64)]


def test_the_tiled_check_admits_the_expected_refused_models(lib):
    assert ADMITTED == [c for c in REFUSED if _tiled_admits(lib, *c)]
    assert len(ADMITTED) == 8


@pytest.mark.parametrize("d,H,layers,hm,lastq", REFUSED)
def test_refused_models_construct_with_tiled_attention_when_the_tiled_check_admits(monkeypatch, lib, d, H, layers, hm,
                                                                                 lastq):
    from rechorus_b200 import plugin
    monkeypatch.setattr(plugin, "_SASREC_LASTQ", lastq)
    admitted = _tiled_admits(lib, d, H, layers, hm, lastq)
    with pytest.raises(ValueError) as e:
        _build(d, H, layers, hm)
    assert ("--tiled_attention 1" in str(e.value)) == admitted
    if admitted:
        m = _build(d, H, layers, hm, tiled=1)
        assert m.tiled_attention and m.p_embeddings.weight.shape == (hm + 1, d)
    else:
        with pytest.raises(ValueError) as e:
            _build(d, H, layers, hm, tiled=1)
        assert "b2r_" in str(e.value)


@pytest.mark.parametrize("d,H,layers,hm", [(64, 4, 2, 200), (64, 1, 2, 200), (64, 4, 1, 512), (128, 4, 2, 150),
                                           (256, 8, 2, 100), (64, 2, 3, 300)])
def test_long_history_models_construct_with_the_flag_only(lib, d, H, layers, hm):
    with pytest.raises(ValueError, match="--tiled_attention 1"):
        _build(d, H, layers, hm)
    assert _build(d, H, layers, hm, tiled=1).tiled_attention


def test_flag_parsing_stand_alone(lib):
    from rechorus_b200 import plugin
    for cls in (plugin.SASRec, plugin.SASRecImpression):
        p = cls.parse_model_args(argparse.ArgumentParser())
        assert p.parse_args([]).tiled_attention == 0
        assert p.parse_args(["--tiled_attention", "1"]).tiled_attention == 1
    assert not _build(64, 4, 2, 50).tiled_attention
    assert not _build(64, 4, 2, 50, tiled=0).tiled_attention


def test_flag_parsing_through_the_overlay(lib):
    import os
    from rechorus_b200 import overlay
    if not os.path.isdir(overlay.DEFAULT_REF):
        pytest.skip("no unmodified reference staged in oracle/_ref (build() without the checkout)")
    classes = overlay.install()
    for name in ("SASRec", "SASRecImpression"):
        p = classes[name].parse_model_args(argparse.ArgumentParser())
        assert p.parse_args([]).tiled_attention == 0
        assert p.parse_args(["--tiled_attention", "1"]).tiled_attention == 1


def test_empty_batch_backward_needs_no_workspace(lib):
    """B = 0 sizes the workspace at 0 bytes, so a NULL workspace is accepted there, as the rt and last-query kernels
    accept an empty batch (no device call is made)"""
    assert lib.b2r_attention_bwd_tiled_workspace_bytes(0, 300, 4) == 0
    p = 256                                                   # any 16-byte aligned address: nothing is dereferenced
    assert lib.b2r_attention_bwd_tiled(p, p, p, 64, None, p, p, p, p, p, p, 64, 0, 300, 64, 4, None, 0, None) == 0
    assert lib.b2r_attention_last_bwd_tiled(p, p, p, 64, p, p, p, p, p, p, 64, 0, 300, 64, 4, None, 0, None) == 0
    assert lib.b2r_attention_bwd_tiled(p, p, p, 64, None, p, p, p, p, p, p, 64, 1, 300, 64, 4, None, 0, None) == -1
