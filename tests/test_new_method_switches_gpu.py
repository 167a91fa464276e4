"""GPU: the outputs of GICP, B200_ICP, FAST_VGICP and B200_VGICP_CUDA are bit-identical under every diagnostic switch their own switch
tests do not set (the BVH build path, the covariance overlap, the index seed, the search and batch copies, stream priorities and the
prefetched covariance kernel's block bound), on clouds that reach the (16, 8) / (8, 16) build shapes and the chained build
(tests/new_method_switch_workload.py, one child process per configuration, four at a time).  The unswitched run is pinned to the
references: one align per method and the k = 49 covariances."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import gicp_pcl_ref as gr
import icp_pcl_ref as ir
import new_method_switch_workload as w
import vgicp_cuda_ref as vc
import vgicp_ref as vr

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

SWITCHES = [
    {"B2R_NO_CLUSTER16": "1"},
    {"B2R_CUB_SORT": "1"},
    {"B2R_NO_COV_OVERLAP": "1"},
    {"B2R_NO_INDEX_SEED": "1"},
    {"B2R_NN_COPIES": "1"},
    {"B2R_NN_COPIES": "2"},
    {"B2R_BATCH_COPIES": "1"},
    {"B2R_BATCH_COPIES": "2"},
    {"B2R_NO_PRIORITY": "1"},
    {"B2R_PREFETCH_PRIORITY": "1"},
    {"B2R_PREFETCH_KNN_BLOCKS": "1"},
]
ALL_SWITCHES = sorted({k for s in SWITCHES for k in s} | {"B2R_NO_PDL", "B2R_SPIN_LIMIT", "B2R_BATCH_CHUNK", "B2R_BATCH_LANES", "B2R_DEBUG_TIMING"})


def label(env):
    return ",".join(f"{k}={v}" for k, v in env.items()) or "baseline"


def run_workload(args):
    extra, out = args
    env = {k: v for k, v in os.environ.items() if k not in ALL_SWITCHES}
    env.update(extra)
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(HERE), HERE] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    try:
        r = subprocess.run([sys.executable, "-s", os.path.join(HERE, "new_method_switch_workload.py"), out], capture_output=True, text=True,
                           env=env, timeout=600)
    except subprocess.TimeoutExpired:
        return {"error": f"{label(extra)}: no result within 600 s"}
    if r.returncode != 0:
        return {"error": f"{label(extra)}: exit {r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"}
    return dict(np.load(out))


@pytest.fixture(scope="module")
def results(tmp_path_factory):
    d = tmp_path_factory.mktemp("new_method_switches")
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


def test_baseline_matches_the_references(results, tmp_path):
    base = results["baseline"]
    assert "error" not in base, base.get("error")
    tgt, src = w.pair(100000, 100)
    # one align per method (the covariance methods fed the engine's covariances, as their own suites do)
    for method in w.METHODS:
        rec = base[f"{method}_align_100000"]
        T, it, conv = rec[:16].reshape(4, 4), int(rec[16]), bool(rec[17])
        assert conv and it >= 1
        if method == "B200_ICP":
            o = ir.Reference(tmp_path).align(src, tgt)
            assert (it, conv) == (o["iterations"], o["converged"]) and np.max(np.abs(T - o["T"])) <= 1e-5
            continue
        _, (scov, tcov) = w.single(method, tgt, src)
        if method == "GICP":
            o = gr.Reference(tmp_path).align(src, tgt, scov=scov, tcov=tcov)
            assert (it, conv) == (o["iterations"], o["converged"])
            gr.end_point_is_as_good(T, o["T"])
        else:
            ref = vr.Reference(tmp_path) if method == "FAST_VGICP" else vc.Reference(tmp_path)
            o = ref.map(tgt, 1.0, tcov).align(src, scov=scov)
            assert (it, conv) == (o["iterations"], o["converged"]) and np.max(np.abs(T - o["T"])) <= 1e-6
    # the k = 49 covariances
    c = w.cov_cloud()
    assert np.max(np.abs(base["GICP_cov_k49"] - gr.Reference(tmp_path).covariances(c, 49))) <= 1e-8
    assert np.max(np.abs(base["FAST_VGICP_cov_k49"] - vr.covariances(c, 49))) <= 1e-8
    assert np.array_equal(base["B200_VGICP_CUDA_cov_k49"], vc.Reference(tmp_path).covariances(c, 49))
