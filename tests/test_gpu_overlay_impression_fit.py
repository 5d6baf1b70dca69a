"""The impression setting's training epochs end to end on an H100: the reference's UNCHANGED ``src/main.py`` runs
BPRMFImpression and SASRecImpression through ``rechorus_b200.overlay`` on the tiny impression dataset of
test_gpu_overlay_impression, with the reference's ImpressionRunner.fit, with ``--device_batches 1`` (training batches built
on the device in the reference DataLoader's own order) and with both ``--device_batches 1 --device_metrics 1``.  The
epoch losses and every dev / test metric line are identical in all three runs.  Skipped only where build() had no
reference to stage."""
import os
import re

import pytest

from tests.test_gpu_overlay_impression import REF, _dataset, _run

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.isfile(os.path.join(REF, "main.py")),
                                 reason="no unmodified reference staged in oracle/_ref (build() without the checkout)")]


@pytest.mark.parametrize("model,extra", [("BPRMF", []),
                                         ("SASRec", ["--history_max", "5", "--num_layers", "1", "--num_heads", "1"])])
def test_device_batches_reproduce_the_reference_fit(tmp_path, model, extra):
    tmp = str(tmp_path)
    _dataset(tmp)
    host_l, host_m, host_out = _run(tmp, "host", model, extra)
    dev_l, dev_m, dev_out = _run(tmp, "device", model, [*extra, "--device_batches", "1"])
    both_l, both_m, both_out = _run(tmp, "both", model, [*extra, "--device_batches", "1", "--device_metrics", "1"])
    # main.py's argument table lists --device_batches only when the runner's parser knows it (B200ImpressionRunner)
    assert re.search(r"device_batches\s*\|\s*1", dev_out) and not re.search(r"device_batches\s*\|", host_out)
    assert len(host_l) == 2 and dev_l == host_l and both_l == host_l
    assert len(host_m) >= 6 and dev_m == host_m and both_m == host_m
