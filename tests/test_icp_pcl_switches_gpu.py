"""GPU: the pcl ICP engine's outputs are bit-identical under every diagnostic switch that changes how its work is enqueued or waited for
(B2R_NO_PDL, B2R_SPIN_LIMIT=1, B2R_BATCH_CHUNK = 1 / 3, B2R_BATCH_LANES=2), each run in a child process."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SWITCHES = ("B2R_NO_PDL", "B2R_SPIN_LIMIT", "B2R_BATCH_CHUNK", "B2R_BATCH_LANES", "B2R_BATCH_COPIES", "B2R_NN_COPIES", "B2R_DEBUG_TIMING")


def run(tmp_path, name, env_extra):
    out = tmp_path / (name + ".npz")
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(env_extra)
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(HERE), HERE] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    subprocess.run([sys.executable, "-s", os.path.join(HERE, "icp_pcl_switch_workload.py"), str(out)], check=True, env=env, timeout=900)
    return dict(np.load(out))


@pytest.fixture(scope="module")
def baseline(tmp_path_factory):
    return run(tmp_path_factory.mktemp("icp_base"), "base", {})


@pytest.mark.parametrize("switch", [{"B2R_NO_PDL": "1"}, {"B2R_SPIN_LIMIT": "1"}, {"B2R_BATCH_CHUNK": "1"}, {"B2R_BATCH_CHUNK": "3"},
                                    {"B2R_BATCH_LANES": "2"}], ids=lambda d: "_".join(f"{k}={v}" for k, v in d.items()))
def test_outputs_are_bit_identical(tmp_path, baseline, switch):
    got = run(tmp_path, "switch", switch)
    assert set(got) == set(baseline)
    for k in baseline:
        assert got[k].dtype == baseline[k].dtype and got[k].tobytes() == baseline[k].tobytes(), k
    assert baseline["batch_false"][:, 17].sum() >= 12 and (baseline["odometry_false"][1:, 17] == 1).all()
