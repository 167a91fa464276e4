"""GPU: pcl ICP (B200_ICP, reciprocal check off and on) and pcl GICP loop batches whose pairs differ in size and in how they end
(tests/mixed_batch_workload.py: sources of 0 to 140 000 points against targets of other sizes, a pair that converges at iteration 1,
pairs stopped by the iteration limit, a pair below the correspondence minimum).  Every record equals a fresh single handle's bit for
bit, the same pair aligned alone and b2r_batch_loop_detect's; iterations, flag and pose match the references; the batch is bit-identical
under B2R_BATCH_CHUNK = 1 / 3 and B2R_BATCH_LANES=2 in child processes.  Then ICP's round prediction on one handle: aligns of very
different length in a row, each equal to a fresh handle, the shortfall topped up."""
import os
import subprocess
import sys

import numpy as np
import pytest

import gicp_pcl_ref as gr
import hdl_graph_slam_b200 as pkg
import icp_pcl_ref as ir
import mixed_batch_workload as mw

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SWITCHES = ("B2R_NO_PDL", "B2R_SPIN_LIMIT", "B2R_BATCH_CHUNK", "B2R_BATCH_LANES", "B2R_BATCH_COPIES", "B2R_NN_COPIES", "B2R_DEBUG_TIMING")
CASES = [("B200_ICP", False), ("B200_ICP", True), ("GICP", False)]


@pytest.fixture(scope="module")
def refs(tmp_path_factory):
    return dict(B200_ICP=ir.Reference(tmp_path_factory.mktemp("icp_pcl_ref")), GICP=gr.Reference(tmp_path_factory.mktemp("gicp_pcl_ref")))


@pytest.fixture(scope="module")
def scene():
    return mw.clouds_and_pairs()


@pytest.fixture(scope="module")
def batches():
    return {case: mw.run_batch(*case) for case in CASES}


def single(method, reciprocal, tgt, src, guess):
    r = pkg.select_registration_method(mw.params(method, reciprocal))
    r.setInputTarget(tgt)
    r.setInputSource(src)
    r.align(guess)
    fit = r.getFitnessScore(2.5) if src.shape[0] else np.finfo(np.float64).max
    out = np.r_[r.getFinalTransformation().astype(np.float64).reshape(-1), r.nr_iterations, r.hasConverged(), fit]
    covs = (r.getCovariances(0, src.shape[0]), r.getCovariances(1, tgt.shape[0])) if method == "GICP" else None
    r.close()
    return out, covs


@pytest.mark.parametrize("method,reciprocal", CASES)
def test_every_record_equals_the_single_handle_and_the_reference(refs, scene, batches, method, reciprocal):
    clouds, pairs = scene
    b = batches[(method, reciprocal)]
    limit = mw.MAX_ITERATIONS[method]
    for i, (s, t, g) in enumerate(pairs):
        want, covs = single(method, reciprocal, clouds[t], clouds[s], g)
        for got in (b["together"][i], b["alone"][i]):
            assert got.tobytes() == want.tobytes(), i
        assert b["loop"][i].tobytes() == np.r_[want[:16], want[17], want[18]].tobytes(), i
        src, tgt = clouds[s], clouds[t]
        T, it, conv = want[:16].reshape(4, 4), int(want[16]), bool(want[17])
        if src.shape[0] == 0:
            assert (it, conv) == (0, False) and np.array_equal(T, g)
            continue
        if method == "B200_ICP":
            # the sequential reciprocal reference takes minutes at 70 000 and 140 000 points: it checks the smaller pairs
            if reciprocal and max(src.shape[0], tgt.shape[0]) > 16384:
                continue
            o = refs[method].align(src, tgt, g, max_iterations=limit, transformation_epsilon=mw.EPSILON[method], reciprocal=reciprocal)
            assert (it, conv) == (o["iterations"], o["converged"]), i
            assert np.max(np.abs(T - o["T"])) <= 1e-5, i
        else:
            scov, tcov = covs
            o = refs[method].align(src, tgt, g, max_iterations=limit, transformation_epsilon=mw.EPSILON[method], scov=scov, tcov=tcov)
            assert (it, conv) == (o["iterations"], o["converged"]), i
            if it == 0:
                assert np.array_equal(T, g)
            elif it < limit:  # converged by the stopping rule (a pair stopped by the limit has no end-point bound)
                gr.end_point_is_as_good(T, o["T"])
    its = b["together"][:, 16]
    conv = b["together"][:, 17]
    sizes = [clouds[s].shape[0] for s, _, _ in pairs]
    assert 1 in its[conv == 1]                                       # the cloud against itself
    assert (its == limit).sum() >= 2                                 # stopped by the iteration limit
    assert its[-1] == 0 and conv[-1] == 0                            # below the correspondence minimum
    assert max(sizes) == 140000 and 0 in sizes


def run_child(tmp_path, name, env_extra):
    out = tmp_path / (name + ".npz")
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update(env_extra)
    env["PYTHONPATH"] = os.pathsep.join([os.path.dirname(HERE), HERE] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    subprocess.run([sys.executable, "-s", os.path.join(HERE, "mixed_batch_workload.py"), str(out)], check=True, env=env, timeout=900)
    return dict(np.load(out))


@pytest.fixture(scope="module")
def child_baseline(tmp_path_factory):
    return run_child(tmp_path_factory.mktemp("mixed_base"), "base", {})


def test_child_baseline_equals_the_in_process_batches(child_baseline, batches):
    for (method, rec), b in batches.items():
        for k, v in b.items():
            assert child_baseline[f"{mw.METHODS[method]}_{int(rec)}_{k}"].tobytes() == v.tobytes(), (method, rec, k)


@pytest.mark.parametrize("switch", [{"B2R_BATCH_CHUNK": "1"}, {"B2R_BATCH_CHUNK": "3"}, {"B2R_BATCH_LANES": "2"}],
                         ids=lambda d: "_".join(f"{k}={v}" for k, v in d.items()))
def test_switches_leave_the_batch_bit_identical(tmp_path, child_baseline, switch):
    got = run_child(tmp_path, "switch", switch)
    assert set(got) == set(child_baseline)
    for k in child_baseline:
        assert got[k].dtype == child_baseline[k].dtype and got[k].tobytes() == child_baseline[k].tobytes(), k


def test_icp_round_prediction_tops_up_short_predictions():
    """one handle aligns pairs needing about 1, 40, 2 and 40 iterations: each equals a fresh handle, and after a short align the next
    long one enqueues its predicted rounds, finds the pair unfinished and tops up (doubling), so it enqueues more rounds than it needed"""
    tgt = gr.scene(16384, seed=140)
    far = gr.pose((1.2, -0.9, 0.1), (0.0, 0.0, 0.12))
    jobs = [(tgt, np.eye(4, dtype=np.float32)), (gr.transform(gr.scene(16384, seed=141), far), np.eye(4, dtype=np.float32)),
            (gr.transform(tgt, gr.pose((0.01, 0.0, 0.0))), np.eye(4, dtype=np.float32)),
            (gr.transform(gr.scene(16384, seed=142), far), np.eye(4, dtype=np.float32))]
    p = {"registration_method": "B200_ICP", "reg_maximum_iterations": "64", "reg_transformation_epsilon": "1e-9"}
    h = pkg.select_registration_method(p)
    h.setInputTarget(tgt)
    its, rounds = [], []
    for src, g in jobs:
        h.setInputSource(src)
        h.getStats(reset=True)
        h.align(g)
        rounds.append(h.getStats()["launches"]["icp_pcl_round"] // 2)
        its.append(h.nr_iterations)
        f = pkg.select_registration_method(p)
        f.setInputTarget(tgt)
        f.setInputSource(src)
        f.align(g)
        assert np.array_equal(h.getFinalTransformation(), f.getFinalTransformation())
        assert (h.nr_iterations, h.hasConverged()) == (f.nr_iterations, f.hasConverged())
        f.close()
    h.close()
    assert its[0] <= 2 and its[2] <= 3 and its[1] >= 20 and its[3] >= 20, its
    for k in (1, 3):  # predicted from the short align before it: topped up past what the pair needed
        assert rounds[k] >= its[k] and rounds[k] > its[k - 1] + 1, (its, rounds)
