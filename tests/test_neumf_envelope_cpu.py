"""CPU: the envelope of NeuMF's fused test_all scorer (b2r_neumf_score_rows_check) against the Linear forward's own route
decision (b2r_linear_fwd_uses_tc), and that decision against the shape class the forward used to test for itself."""
import pytest


@pytest.fixture(scope="module")
def ops():
    from rechorus_b200 import build
    build.build()
    from rechorus_b200 import ops
    return ops


def _forward_all_tc(ops, d, layers, M):
    """every hidden layer of NeuMF's forward on a batch of M candidate rows runs on the tensor-core Linear"""
    K = 2 * d
    for N in layers:
        if not ops.linear_fwd_uses_tc(M, N, K):
            return False
        K = N
    return True


# (d, layers, Bn, n_items, fused)
CASES = [
    (32, [32, 16], 7, 3001, True),
    (32, [64, 32], 3, 20011, True),
    (64, [64], 1, 4096, True),
    (64, [64, 32, 16], 256, 1_000_000, True),
    (64, [64], 1, 4095, False),                # below the forward's tensor-core threshold
    (32, [32, 16], 64, 64, True),
    (32, [32, 16], 65, 63, False),             # 4095 candidate rows
    (128, [10], 64, 2000, False),              # d outside {32, 64}; N = 10 is the SGEMM's
    (16, [32], 64, 2000, False),               # K = 32 is on the tensor cores, d = 16 is not the scorer's
    (32, [48, 32], 64, 2000, False),           # second layer K = 48: the forward's SGEMM
    (32, [48], 64, 2000, True),                # N = 48 runs at wgmma width 64
    (64, [48], 64, 2000, True),
    (32, [128, 32], 64, 2000, True),
    (32, [96, 16], 64, 2000, True),            # K = 96 (three 32-float slabs) in a later layer
    (32, [96, 32], 64, 2000, True),
    (32, [32, 96, 16], 64, 2000, True),
    (32, [96, 96, 16], 64, 2000, False),       # 274 KB: two 128-wide W tiles
    (64, [64, 96], 64, 2000, False),           # N = 96 runs at wgmma width 128: registers at d = 64
    (32, [128, 64], 64, 2000, False),          # 242 KB of resident weights and operands
    (64, [128], 64, 2000, False),              # registers at d = 64
    (64, [128, 128], 64, 2000, False),
    (32, [128, 128, 128], 64, 2000, False),    # W tiles beyond one CTA's shared memory
    (32, [256], 64, 2000, False),              # on the tensor cores (K = 64), wider than the scorer's accumulator
    (64, [256], 64, 2000, False),              # N > 128 with K > 64: the forward's SGEMM
    (32, [32, 32, 32, 32], 64, 2000, True),
    (32, [32, 32, 32, 32, 32], 64, 2000, False),
    (32, [], 64, 2000, False),
    (32, [32], 1 << 16, 1 << 15, False),       # 2^31 rows
]


@pytest.mark.parametrize("d,layers,Bn,n_items,fused", CASES)
def test_envelope_table(ops, d, layers, Bn, n_items, fused):
    err = ops.neumf_all_items_error(d, layers, Bn, n_items)
    assert (err is None) == fused, err
    if fused:                                  # inside the envelope the forward runs every layer on the tensor cores
        assert d in (32, 64) and _forward_all_tc(ops, d, layers, Bn * n_items)
    if layers and d in (32, 64) and 4096 <= Bn * n_items < 2 ** 31 and not _forward_all_tc(ops, d, layers, Bn * n_items):
        assert err is not None and "tensor-core" in err


def test_linear_route_decision_matches_the_forwards_former_condition(ops):
    for M in (1, 4095, 4096, 1 << 20):
        for K in (16, 24, 32, 48, 64, 96, 128, 160, 256):
            for N in (1, 8, 16, 32, 48, 64, 128, 144, 256, 272):
                old = M >= 4096 and K % 32 == 0 and K <= 128 and N % 16 == 0 and N <= 256
                refused = N > 128 and K > 64      # the C side refused these and the forward fell back to the SGEMM
                assert ops.linear_fwd_uses_tc(M, N, K) == (old and not refused), (M, N, K)


def test_window_rows_bound_the_score_block(ops):
    assert ops.neumf_window_rows(256, 1_000_000) == 8
    assert ops.neumf_window_rows(256, 100_000) == 83
    assert ops.neumf_window_rows(32, 2000) == 32
    assert ops.neumf_window_rows(256, 50_000_000) == 1
    for Bn, n in ((1, 10), (256, 1_000_000), (7, 3001), (3, 20_000_000)):
        r = ops.neumf_window_rows(Bn, n)
        assert 1 <= r <= Bn and (r == 1 or r * n * 4 <= 32 << 20)
