"""Generate tests/golden/overlay_reference.npz: the UNMODIFIED reference's own CPU runs of the command lines
tests/test_gpu_overlay.py drives through the overlay (per-epoch losses, the Test metric line, the final checkpoint).

Run where build() has staged the reference in oracle/_ref (oracle/stage_reference.py):
    python tests/golden/make_overlay_golden.py
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import test_gpu_overlay as T  # noqa: E402


def main():
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        T._dataset(tmp)
        for tag, (model, flags) in T.REFERENCE_RUNS.items():
            losses, metrics, weights, _ = T._run(tmp, tag, T.REFERENCE, model, flags, "")
            out[tag + "/losses"] = np.asarray(losses, dtype=np.float64)
            for k, v in metrics.items():
                out[tag + "/metric/" + k] = np.float64(v)
            for k, v in weights.items():
                out[tag + "/w/" + k] = v.detach().cpu().numpy()
            print(tag, losses, metrics)
    np.savez_compressed(T.GOLDEN, **out)
    print(T.GOLDEN, os.path.getsize(T.GOLDEN), "bytes")


if __name__ == "__main__":
    main()
