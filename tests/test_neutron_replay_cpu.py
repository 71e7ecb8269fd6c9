"""tools/neutron_replay.py end to end on the emulated device (tests/emulated_device.py with the NeutronNova entries
of tests/emulated_neutron.py): the tool's Neutron and Nova folds, timings and --check path (restated verify, C-oracle
is_sat sum, tampered T, Nova's is_sat_relaxed) run without a GPU."""
import gc
import os
import sys

import emulated_neutron

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_neutron_replay_check_on_the_emulated_device(oracle):
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import neutron_replay
    emulated_neutron.install()
    try:
        out = neutron_replay.run(log2n=8, reps=1, check_proof=True)
        assert out["check"] is True, out
        assert out["neutron_ms"]["total"] > 0 and out["nova_ms"] > 0
        assert (out["left"], out["right"], out["comm_E_points"]) == (16, 16, 32)
    finally:
        gc.collect()
        emulated_neutron.uninstall()
