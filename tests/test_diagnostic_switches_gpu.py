"""Every diagnostic environment switch leaves every output bit-identical (README, "Environment switches").

The engine reads its switches once per process, so each configuration runs tests/switch_workload.py in a fresh child process:
GICP odometry with and without the next frame announced and with the voxel-grid downsample, a single GICP pair, k-NN and
covariances on a 100 000-point target, the voxel grid and the prefilter (each outlier method) on a KITTI-size scan, NDT
derivative / Hessian passes and aligns on a 131 072-point source, a 16-pair GICP batch with loop detection and fitness scores,
an NDT batch of mixed sizes, and the same passes, aligns (both line-search polarities) and batch for the pcl NDT method.
Each configuration's SHA-1 per output must equal the baseline's (no switch set), and the baseline itself is pinned to the oracle: its single GICP pair and first odometry step to oracle.gicp_align, its NDT derivatives
to the oracle's derivative pass, its pcl NDT derivatives to tests/ndt_pcl_ref.cpp."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
from common import rot_err, trans_err, relrel
from ndt_pcl_ref import Reference
from switch_workload import NDT_P, sha

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SWITCHES = [
    {"B2R_NO_PDL": "1"},
    {"B2R_NO_INDEX_SEED": "1"},
    {"B2R_NO_PRIORITY": "1"},
    {"B2R_PREFETCH_PRIORITY": "1"},
    {"B2R_PREFETCH_KNN_BLOCKS": "1"},
    {"B2R_PREFETCH_KNN_BLOCKS": "2"},
    {"B2R_PREFETCH_KNN_BLOCKS": "3"},
    {"B2R_SPIN_LIMIT": "1"},            # every wait takes the blocking fallback
    {"B2R_NO_COV_OVERLAP": "1"},
    {"B2R_NN_COPIES": "1"},
    {"B2R_NN_COPIES": "2"},
    {"B2R_BATCH_LANES": "2"},
    {"B2R_BATCH_CHUNK": "1"},
    {"B2R_BATCH_CHUNK": "3"},
    {"B2R_NDT_WAVES": "0.01"},
    {"B2R_NDT_WAVES": "0.5"},
    {"B2R_NDT_WAVES": "3"},
    {"B2R_NO_CLUSTER16": "1"},
    {"B2R_CUB_SORT": "1"},
    {"B2R_DEBUG_TIMING": "1"},
]
ALL_SWITCHES = sorted({k for s in SWITCHES for k in s} | {"B2R_BATCH_COPIES"})


def label(env):
    return ",".join(f"{k}={v}" for k, v in env.items()) or "baseline"


def run_workload(extra):
    env = {k: v for k, v in os.environ.items() if k not in ALL_SWITCHES}
    env.update(extra)
    try:
        r = subprocess.run([sys.executable, os.path.join(HERE, "switch_workload.py")], capture_output=True, text=True, env=env, timeout=600, cwd=ROOT)
    except subprocess.TimeoutExpired:
        return {"error": f"{label(extra)}: no result within 600 s"}
    if r.returncode != 0:
        return {"error": f"{label(extra)}: exit {r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"}
    return json.loads(r.stdout.strip().splitlines()[-1])  # B2R_DEBUG_TIMING prints before it


@pytest.fixture(scope="module")
def results():
    """every configuration, four child processes at a time (the outputs may not depend on what else runs on the device)"""
    confs = [{}] + SWITCHES
    with ThreadPoolExecutor(max_workers=4) as ex:
        outs = list(ex.map(run_workload, confs))
    return {label(c): o for c, o in zip(confs, outs)}


def test_baseline_matches_the_oracle(results, synth, oracle, tmp_path):
    assert "error" not in results["baseline"], results["baseline"].get("error")
    a = results["baseline"]["anchor"]
    f0, f1 = synth.scan("vlp16", frame=0, stride=8), synth.scan("vlp16", frame=1, stride=8)
    o = oracle.gicp_align(f1, f0, np.eye(4, dtype=np.float32))
    T = np.array(a["gicp_T"])
    assert trans_err(T, o["T"]) < 1e-6 and rot_err(T, o["T"]) < 1e-6 and a["gicp_iterations"] == o["iterations"]
    assert a["gicp_corr"] == sha(np.asarray(o["corr"], np.int32))
    # the odometry's first step registers frame 1 against keyframe 0 from the identity
    T1 = np.array(a["odometry_trans1"])
    assert trans_err(T1, o["T"]) < 1e-6 and rot_err(T1, o["T"]) < 1e-6 and a["odometry_iterations1"] == o["iterations"]
    src, tgt = synth.scan("hdl32e", frame=1, stride=8), synth.scan("hdl32e", frame=0, stride=8)
    od = oracle.NdtMap(tgt, 1.0).derivatives(src, NDT_P, search_method=7)
    n = a["ndt"]
    assert n["npairs"] == od["n_pairs"] > 10000
    assert abs(n["score"] - od["score"]) <= 1e-9 * abs(od["score"])
    assert relrel(n["g"], od["g"]) < 1e-9 and relrel(n["H"], od["H"]) < 1e-9
    # the pcl NDT passes at the same pose, against the sequential reference of that method (tests/ndt_pcl_ref.cpp)
    op = Reference(tmp_path).map(tgt, 1.0).derivatives(src, NDT_P)
    n = a["ndt_pcl"]
    assert n["npairs"] == op["n_pairs"] > 10000
    assert abs(n["score"] - op["score"]) <= 1e-9 * abs(op["score"])
    assert relrel(n["g"], op["g"]) < 1e-9 and relrel(n["H"], op["H"]) < 1e-9


@pytest.mark.parametrize("env", SWITCHES, ids=label)
def test_switch_leaves_every_output_unchanged(results, env):
    assert "error" not in results["baseline"], results["baseline"].get("error")
    assert "error" not in results[label(env)], results[label(env)].get("error")
    base = results["baseline"]["outputs"]
    got = results[label(env)]["outputs"]
    assert got.keys() == base.keys()
    differ = [k for k in base if got[k] != base[k]]
    assert not differ, f"{label(env)} changes {differ}"
