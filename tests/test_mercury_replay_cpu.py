"""tools/mercury_replay.py end to end on the emulated device (tests/emulated_device.py with
the Mercury entries of tests/emulated_mercury.py): the tool's prover call,
timings and --check path (restated verifier, C by the C oracle) run without a GPU."""
import gc
import os
import sys

import emulated_mercury

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_mercury_replay_check_on_the_emulated_device(oracle):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import mercury_replay
    emulated_mercury.install()
    try:
        for log2n in (8, 7):
            out = mercury_replay.run(log2n=log2n, reps=1, check_proof=True)
            assert out["check"] is True, out
            assert out["ms"]["total"] > 0 and out["msm_points"] > (1 << log2n)
    finally:
        gc.collect()
        emulated_mercury.uninstall()
