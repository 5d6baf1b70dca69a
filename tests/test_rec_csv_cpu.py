"""CPU: the text save_rec_results' device writer produces, pinned against NumPy and pandas without a GPU.

The formatter (rechorus_b200/csrc/rec_format.cuh) is compiled for the host (tests/rec_format_harness.cu) and compared
with NumPy's repr on the designed sample of 10^7 float32 bit patterns in both element styles, on int64 edges, and at the
adjacent pairs around the notation switch points.  The route predicate (runner.rec_csv_style) and the argument checks of
b2r_rec_csv are checked too."""
import os
import re

import numpy as np
import pytest

from tests import rec_csv_oracle as O

pytestmark = pytest.mark.skipif(not os.path.exists(O.NVCC), reason="nvcc is needed to build the host harness")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return O.build_harness(str(tmp_path_factory.mktemp("rec_harness")))


@pytest.fixture(scope="module")
def sample():
    return O.designed_sample()


@pytest.mark.parametrize("style", [O.STYLE_NP, O.STYLE_BARE])
def test_float32_text_equals_numpy_repr_on_the_designed_sample(exe, sample, style, tmp_path):
    assert sample.size >= 10_000_000
    got = O.harness(exe, sample, style, str(tmp_path))
    want = O.numpy_repr(sample, style)
    assert len(got) == len(want) == sample.size
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    assert not bad, [(hex(int(sample[i])), got[i], want[i]) for i in bad[:10]]
    longest = max(len(t) for t in got)
    assert longest <= (31 if style == O.STYLE_NP else 19)          # recfmt::row_bytes_max's per-element bound


@pytest.mark.parametrize("style", [O.STYLE_NP, O.STYLE_BARE])
def test_int64_text_equals_numpy_repr(exe, style, tmp_path):
    v = O.int64_sample()
    got = O.harness(exe, v, style, str(tmp_path), ints=True)
    assert got == O.numpy_repr(v, style, ints=True)
    assert max(len(t) for t in got) == (30 if style == O.STYLE_NP else 20)


def _bits(x):
    return int(np.float32(x).view(np.uint32))


SWITCHES = {  # (last float32 on one side, first on the other): scientific below 1e-4, and at or above hi
    "1e-4": (0x38d1b717, 0x38d1b718),
    "1e6": (_bits(999999.94), _bits(1e6)),
    "1e16": (_bits(1e16) - 1, _bits(1e16)),
}


@pytest.mark.parametrize("style", [O.STYLE_NP, O.STYLE_BARE])
def test_notation_switch_points_and_observed_texts(exe, style, tmp_path):
    pairs = np.array([b for p in SWITCHES.values() for b in p], dtype=np.uint32)
    pairs = np.concatenate([pairs, pairs | 0x80000000])
    got = O.harness(exe, pairs, style, str(tmp_path))
    assert got == O.numpy_repr(pairs, style)
    bare = [re.sub(r"^np\.float32\((.*)\)$", r"\1", t) for t in got]
    assert bare[:2] == ["1e-04", "0.000100000005"]
    if style == O.STYLE_NP:
        assert bare[2:6] == ["999999.94", "1e+06", "9.999999e+15", "1e+16"]
    else:
        assert bare[2:6] == ["999999.94", "1000000.0", "9999999000000000.0", "1e+16"]
    assert bare[6:8] == ["-1e-04", "-0.000100000005"]
    specials = np.array([0, 0x80000000, 0x7f800000, 0xff800000, 0x7fc00000, 0xffc00001, 0x7f800001, 1, 0x7f7fffff,
                         _bits(1e7), _bits(2.0 ** 24), _bits(1048576.0), _bits(0.3), _bits(100000.0)], dtype=np.uint32)
    got = O.harness(exe, specials, style, str(tmp_path))
    assert got == O.numpy_repr(specials, style)
    big = ["1e+07", "1.6777216e+07", "1.048576e+06"] if style == O.STYLE_NP else ["10000000.0", "16777216.0", "1048576.0"]
    assert [re.sub(r"^np\.float32\((.*)\)$", r"\1", t) for t in got] == \
        ["0.0", "-0.0", "inf", "-inf", "nan", "nan", "nan", "1e-45", "3.4028235e+38", *big, "0.3", "100000.0"]


def test_power_of_five_tables_match_their_definition():
    """the two tables of rec_format.cuh are floor(2^(pow5bits(i) - 1 + 59) / 5^i) + 1 and floor(5^i / 2^(pow5bits(i) - 61))"""
    src = open(os.path.join(O.ROOT, "rechorus_b200", "csrc", "rec_format.cuh")).read()

    def table(name):
        body = re.search(r"#define %s \{(.*?)\}" % name, src, re.S).group(1)
        return [int(x, 16) for x in re.findall(r"0x([0-9a-f]+)ull", body)]

    def pow5bits(e):
        return ((e * 1217359) >> 19) + 1

    inv, pw = table("B2R_POW5_INV_SPLIT"), table("B2R_POW5_SPLIT")
    assert inv == [(1 << (pow5bits(i) - 1 + 59)) // 5 ** i + 1 for i in range(31)]
    assert pw == [(5 ** i << 61) >> pow5bits(i) for i in range(48)]
    assert all(pow5bits(i) == (5 ** i).bit_length() for i in range(1, 48))


# ---- the route: when the device writes save_rec_results' CSV -----------------------------------------------------

def test_route_follows_numpy_printing_separator_and_user_ids():
    from rechorus_b200 import ops
    from rechorus_b200.runner import rec_csv_style
    users = np.arange(1, 5, dtype=np.int64)
    for sep in ("\t", ",", " ", ";", "1", "e", "|", "["):
        assert rec_csv_style(sep, users) == ops.REC_STYLE_NP
        assert rec_csv_style(sep, list(users)) == ops.REC_STYLE_NP
    with np.printoptions(legacy="1.25"):
        assert rec_csv_style("\t", users) == ops.REC_STYLE_BARE
    for legacy in ("1.13", "1.21"):
        with np.printoptions(legacy=legacy):
            assert rec_csv_style("\t", users) is None
    for sep in ("", "\t\t", "::", '"', "\r", "\n", "\0", "é", b",", None):
        assert rec_csv_style(sep, users) is None, sep
    assert rec_csv_style("\t", ["a", "b"]) is None
    assert rec_csv_style("\t", np.array([0.5, 1.5])) is None
    assert rec_csv_style("\t", np.array([2 ** 63], dtype=np.uint64)) is None
    assert rec_csv_style("\t", np.array([3], dtype=np.uint32)) == ops.REC_STYLE_NP
    assert rec_csv_style("\t", []) == ops.REC_STYLE_NP                 # an empty phase: the header alone


def test_rec_csv_entry_rejects_bad_arguments_without_a_gpu():
    from rechorus_b200 import build
    build.build()
    from rechorus_b200 import lib as L
    h = L.load()
    fake = 256                                                        # never dereferenced: the checks come first
    for sep in (0, ord('"'), ord("\r"), ord("\n"), 200):
        assert h.b2r_rec_csv(fake, fake, fake, 4, 10, 0, sep, fake, 1 << 20, fake, fake, 1 << 20, None) == -1
    assert b"sep" in h.b2r_last_error()
    assert h.b2r_rec_csv(fake, fake, fake, 4, 10, 2, 9, fake, 1 << 20, fake, fake, 1 << 20, None) == -1
    assert h.b2r_rec_csv(None, fake, fake, 4, 10, 0, 9, fake, 1 << 20, fake, fake, 1 << 20, None) == -1
    need = h.b2r_rec_csv_text_bytes_max(4, 10, 0)
    assert need == 4 * ((20 + 2) + 1 + (2 + 18 + 300 + 2) + 1 + (2 + 18 + 310 + 2) + 1)
    assert h.b2r_rec_csv(fake, fake, fake, 4, 10, 0, 9, fake, need - 1, fake, fake, 1 << 20, None) == -2
    assert h.b2r_rec_csv_text_bytes_max(-1, 10, 0) == 0 and h.b2r_rec_csv_text_bytes_max(4, 10, 5) == 0
