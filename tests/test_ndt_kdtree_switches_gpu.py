"""GPU: every diagnostic switch that reaches the NDT_OMP KDTREE paths leaves their outputs bit-identical.  Each configuration runs
tests/ndt_kdtree_switch_workload.py in a fresh child process (the engine reads its switches once per process): B2R_NDT_WAVES = 0.01 / 0.5 / 3,
B2R_NO_PDL, B2R_SPIN_LIMIT=1, B2R_BATCH_CHUNK = 1 / 3, B2R_BATCH_LANES=2, B2R_CUB_SORT and B2R_NO_CLUSTER16.  The unswitched run is pinned
to tests/ndt_kdtree_ref.cpp, and its single-rank b2r_batch_loop_detect records to b2r_batch_align's."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from hdl_graph_slam_b200 import synth
import ndt_kdtree_switch_workload as w
from ndt_kdtree_ref import Reference

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SWITCHES = [{"B2R_NDT_WAVES": "0.01"}, {"B2R_NDT_WAVES": "0.5"}, {"B2R_NDT_WAVES": "3"}, {"B2R_NO_PDL": "1"}, {"B2R_SPIN_LIMIT": "1"},
            {"B2R_BATCH_CHUNK": "1"}, {"B2R_BATCH_CHUNK": "3"}, {"B2R_BATCH_LANES": "2"}, {"B2R_CUB_SORT": "1"}, {"B2R_NO_CLUSTER16": "1"}]
ALL_SWITCHES = sorted({k for s in SWITCHES for k in s} | {"B2R_DEBUG_TIMING", "B2R_NO_COV_OVERLAP", "B2R_NO_INDEX_SEED", "B2R_NN_COPIES"})


def label(env):
    return ",".join(f"{k}={v}" for k, v in env.items()) or "baseline"


def run_workload(args):
    extra, out = args
    env = {k: v for k, v in os.environ.items() if k not in ALL_SWITCHES}
    env.update(extra)
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(HERE), HERE] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    try:
        r = subprocess.run([sys.executable, "-s", os.path.join(HERE, "ndt_kdtree_switch_workload.py"), out], capture_output=True, text=True,
                           env=env, timeout=900)
    except subprocess.TimeoutExpired:
        return {"error": f"{label(extra)}: no result within 900 s"}
    if r.returncode != 0:
        return {"error": f"{label(extra)}: exit {r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"}
    return dict(np.load(out))


@pytest.fixture(scope="module")
def results(tmp_path_factory):
    d = tmp_path_factory.mktemp("ndt_kdtree_switches")
    confs = [{}] + SWITCHES
    with ThreadPoolExecutor(max_workers=4) as ex:
        outs = list(ex.map(run_workload, [(c, str(d / f"run{i}.npz")) for i, c in enumerate(confs)]))
    return {label(c): o for c, o in zip(confs, outs)}


@pytest.mark.parametrize("switch", SWITCHES, ids=label)
def test_outputs_are_bit_identical(results, switch):
    base, got = results["baseline"], results[label(switch)]
    assert "error" not in base, base.get("error")
    assert "error" not in got, got.get("error")
    assert set(got) == set(base)
    for k in base:
        assert got[k].dtype == base[k].dtype and got[k].tobytes() == base[k].tobytes(), k


def test_baseline_matches_the_reference(results, tmp_path):
    base = results["baseline"]
    assert "error" not in base, base.get("error")
    tgt, src = synth.scan("hdl32e", frame=0, stride=8), synth.scan("hdl32e", frame=1, stride=8)
    M = Reference(tmp_path).map(tgt, 1.0)
    o = M.derivatives(src, w.POSE)
    d = base["deriv"]
    assert d[-1] == o["n_pairs"] > 0
    assert abs(d[0] - o["score"]) <= 1e-9 * abs(o["score"])
    assert np.max(np.abs(d[1:7] - o["g"])) <= 1e-9 * np.max(np.abs(o["g"]))
    assert np.max(np.abs(d[7:43] - o["H"].reshape(-1))) <= 1e-9 * np.max(np.abs(o["H"]))
    Hh = M.hessian_at(src, w.POSE).reshape(-1)
    assert np.max(np.abs(base["hess"] - Hh)) <= 1e-9 * np.max(np.abs(Hh))
    a = M.align(src, mt_interval_flag=1)
    rec = base["align"]
    assert (int(rec[16]), bool(rec[17])) == (a["iterations"], a["converged"])
    assert np.max(np.abs(rec[:16].reshape(4, 4) - a["T"])) < 1e-4
    assert base["loop_align"].tobytes() == base["loop_detect"].tobytes()
