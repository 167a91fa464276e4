"""GPU: b2r_floor_detect's outputs are bitwise the same under the batch-size switch and the BVH-build / launch switches it runs
through (each run in a child process: the switches are read once per process)."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SWITCHES = [{}, {"B2R_FLOOR_HYPOTHESES": "1"}, {"B2R_FLOOR_HYPOTHESES": "7"}, {"B2R_FLOOR_HYPOTHESES": "1000"}, {"B2R_CUB_SORT": "1"},
            {"B2R_NO_CLUSTER16": "1"}, {"B2R_NO_PDL": "1"}]


def _run(tmp_path, env_extra):
    path = str(tmp_path / ("out_" + "_".join(f"{k}{v}" for k, v in env_extra.items()) + ".npz"))
    env = dict(os.environ, **env_extra)
    env["PYTHONPATH"] = os.pathsep.join([HERE, os.path.dirname(HERE)] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    subprocess.check_call([sys.executable, "-s", os.path.join(HERE, "floor_switch_workload.py"), path], env=env)
    return np.load(path)


@pytest.fixture(scope="module")
def baseline(tmp_path_factory):
    return _run(tmp_path_factory.mktemp("floor_sw"), {})


@pytest.mark.parametrize("switch", SWITCHES[1:], ids=lambda s: ",".join(f"{k}={v}" for k, v in s.items()))
def test_switch_gives_identical_outputs(tmp_path, baseline, switch):
    got = _run(tmp_path, switch)
    assert sorted(got.files) == sorted(baseline.files)
    for k in baseline.files:
        a, b = baseline[k], got[k]
        if a.dtype == np.float32:
            a, b = a.view(np.uint32), b.view(np.uint32)
        assert np.array_equal(a, b), k
