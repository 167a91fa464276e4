"""GPU: every diagnostic switch that reaches the pclomp GICP paths leaves their outputs bit-identical.  Each configuration runs
tests/gicp_omp_switch_workload.py in a fresh child process (the engine reads its switches once per process): the switches of
tests/test_new_method_switches_gpu.py plus B2R_NO_PDL, B2R_SPIN_LIMIT=1, B2R_BATCH_CHUNK = 1 / 3 and B2R_BATCH_LANES=2.  The unswitched
run is pinned to tests/gicp_omp_ref.cpp, and its single-rank b2r_batch_loop_detect records to b2r_batch_align's."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import gicp_omp_ref as gor
import gicp_omp_switch_workload as w
import gicp_pcl_ref as gr
from test_new_method_switches_gpu import SWITCHES as NEW_METHOD_SWITCHES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SWITCHES = NEW_METHOD_SWITCHES + [{"B2R_NO_PDL": "1"}, {"B2R_SPIN_LIMIT": "1"}, {"B2R_BATCH_CHUNK": "1"}, {"B2R_BATCH_CHUNK": "3"},
                                  {"B2R_BATCH_LANES": "2"}]
ALL_SWITCHES = sorted({k for s in SWITCHES for k in s} | {"B2R_DEBUG_TIMING"})


def label(env):
    return ",".join(f"{k}={v}" for k, v in env.items()) or "baseline"


def run_workload(args):
    extra, out = args
    env = {k: v for k, v in os.environ.items() if k not in ALL_SWITCHES}
    env.update(extra)
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(HERE), HERE] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    try:
        r = subprocess.run([sys.executable, "-s", os.path.join(HERE, "gicp_omp_switch_workload.py"), out], capture_output=True, text=True,
                           env=env, timeout=900)
    except subprocess.TimeoutExpired:
        return {"error": f"{label(extra)}: no result within 900 s"}
    if r.returncode != 0:
        return {"error": f"{label(extra)}: exit {r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"}
    return dict(np.load(out))


@pytest.fixture(scope="module")
def results(tmp_path_factory):
    d = tmp_path_factory.mktemp("gicp_omp_switches")
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
    ref = gor.Reference(tmp_path)
    tgt, src = w.pair(100000, 100)
    rec = base["align_100000"]
    T, it, conv = rec[:16].reshape(4, 4), int(rec[16]), bool(rec[17])
    _, (scov, tcov) = w.single(tgt, src)
    o = ref.align(src, tgt, w.GUESS, scov=scov, tcov=tcov)
    assert conv and it >= 1 and (it, conv) == (o["iterations"], o["converged"])
    gr.end_point_is_as_good(T, o["T"])
    assert np.max(np.abs(base["cov_k49"] - ref.covariances(w.scene(16384, seed=120), 49))) <= 1e-8
    assert base["loop_align"].tobytes() == base["loop_detect"].tobytes()
