"""GPU: every diagnostic switch that reaches the FastVGICPCuda (B200_VGICP_CUDA) paths leaves their outputs bit-identical.  Each configuration runs
tests/vgicp_cuda_switch_workload.py in a fresh child process (the engine reads its switches once per process): a FastVGICPCuda odometry chain with
the next frame announced, and a 24-pair loop batch with fitness through b2r_batch_align and the single-rank b2r_batch_loop_detect
(24 pairs: the batch really splits over two lanes under B2R_BATCH_LANES=2; B2R_BATCH_CHUNK=1 / 3 runs it in several chunks)."""
import json
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SWITCHES = [{"B2R_NO_PDL": "1"}, {"B2R_SPIN_LIMIT": "1"}, {"B2R_BATCH_CHUNK": "1"}, {"B2R_BATCH_CHUNK": "3"}, {"B2R_BATCH_LANES": "2"}]
ALL = sorted({k for s in SWITCHES for k in s} | {"B2R_BATCH_COPIES", "B2R_NN_COPIES", "B2R_DEBUG_TIMING"})


def label(env):
    return ",".join(f"{k}={v}" for k, v in env.items()) or "baseline"


def run_workload(extra):
    env = {k: v for k, v in os.environ.items() if k not in ALL}
    env.update(extra)
    try:
        r = subprocess.run([sys.executable, os.path.join(HERE, "vgicp_cuda_switch_workload.py")], capture_output=True, text=True, env=env, timeout=600,
                           cwd=ROOT)
    except subprocess.TimeoutExpired:
        return {"error": f"{label(extra)}: no result within 600 s"}
    if r.returncode != 0:
        return {"error": f"{label(extra)}: exit {r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"}
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.fixture(scope="module")
def results():
    confs = [{}] + SWITCHES
    with ThreadPoolExecutor(max_workers=3) as ex:
        outs = list(ex.map(run_workload, confs))
    return {label(c): o for c, o in zip(confs, outs)}


def test_baseline_loop_detect_equals_batch_align_and_argmin(results):
    """one rank: b2r_batch_loop_detect's records are b2r_batch_align's, and its choice per group is LoopDetector::matching's
    (best converged fitness, a later equal score wins, none above the threshold; loop_detector.hpp:147,160-163)"""
    b = results["baseline"]
    assert "error" not in b, b.get("error")
    a, d = np.array(b["batch_align"], np.uint64), np.array(b["loop_detect"], np.uint64)
    assert np.array_equal(a, d)
    gf = b["group_first"]
    fit = np.ascontiguousarray(a[:, 16]).view(np.float64)
    conv = a[:, 17] != 0
    assert np.isfinite(fit).all() and conv.any()
    for g in range(len(gf) - 1):
        best, best_score = -1, np.finfo(np.float64).max
        for i in range(gf[g], gf[g + 1]):
            if conv[i] and not fit[i] > best_score:
                best, best_score = i - gf[g], fit[i]
        assert b["best"][g] == (best if best_score <= 0.5 else -1)


@pytest.mark.parametrize("conf", SWITCHES, ids=label)
def test_switch_leaves_vgicp_cuda_outputs_unchanged(results, conf):
    base, got = results["baseline"], results[label(conf)]
    assert "error" not in base, base.get("error")
    assert "error" not in got, got.get("error")
    assert got["outputs"] == base["outputs"]
