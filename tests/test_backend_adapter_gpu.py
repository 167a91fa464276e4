"""GPU: the back-end drop-in (adapter/b200_backend.hpp) EXECUTED through tests/backend_harness.cpp and the test-only stand-ins
adapter/pcl_shim.hpp + adapter/backend_shim.hpp, the way hdl_graph_slam_nodelet drives LoopDetector, InformationMatrixCalculator and
MapCloudGenerator (apps/hdl_graph_slam_nodelet.cpp:235,528,549-577), all three on one shared keyframe cache.

A session of optimisation ticks over the synthetic loop trajectory: new keyframes each tick, graph estimates moved between ticks, a tick
without candidates, a loop that gates out a later new keyframe of the same tick, and one empty keyframe cloud.  For FAST_GICP and the
factory default NDT_OMP:
  - detect() registers the loops of the reference's walk (loop_detector.hpp:57-171) restated on one handle, relative poses bitwise, and
    last_edge_accum_distance after every tick;
  - calc_information_matrix is bitwise b2r_information_from_fitness of b2r_fitness on a fresh handle, its score within the suite's
    tolerance of the oracle's calc_fitness_score, use_const_inf_matrix and the no-neighbour case (DBL_MAX) included;
  - generate() is bitwise b2r_map_cloud_generate on the same clouds and poses, and nullptr without keyframes;
  - every keyframe cloud is uploaded exactly once in the session: a second pass over the same calls uploads no point;
  - generate() on a second thread while detect() and the information matrices run gives the serial answers."""
import os
import struct
import subprocess
import numpy as np
import pytest
import torch  # noqa: F401  before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from common import perturb
from test_loop_gate import ref_find_candidates

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DBL_MAX = np.finfo(np.float64).max
KEYFRAME, ESTIMATE, DETECT, INFO, MAP = 1, 2, 3, 4, 5
EMPTY = "empty"
# (trajectory frame of the cloud, accumulated distance, trajectory frame of the estimate) per new keyframe, one list per tick
TICKS = [
    [(0, 0.0, 0), (2, 2.0, 2), (10, 10.0, 10), (12, 12.0, 12)],  # nothing registered yet
    [(20, 20.0, 20), (120, 120.0, 120), (EMPTY, 140.0, 24)],  # keyframes registered, no candidate
    [(251, 251.0, 251), (253, 253.0, 253), (261, 261.0, 261), (271, 271.0, 271)],  # 251's loop gates 253; the empty cloud is a candidate of 271
    [(276, 276.0, 276), (300, 300.0, 300)],
]
MAP_RES = [0.05, 0.0, 0.05, -1.0, 0.05]  # before each tick's detect, and once after the last tick
CONFIGS = {"gicp": {"registration_method": "FAST_GICP"}, "ndt_omp": {"reg_resolution": "1.0"}}  # NDT_OMP: the factory default
LOOP_PARAMS = dict(distance_thresh=5.0, accum_distance_thresh=8.0, min_edge_interval=5.0)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    from hdl_graph_slam_b200 import build
    build.build_engine()
    exe = str(tmp_path_factory.mktemp("backend") / "backend_harness")
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++14", "-O1", "-Wall", "-pthread",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", exe,
                           os.path.join(ROOT, "tests", "backend_harness.cpp"), "-L", lib, "-lb200reg", "-Wl,-rpath," + lib])
    return exe


def session(synth):
    """the clouds (the empty one last) and the operation list: (op, fields...).  Keyframe k of the test = the k-th KEYFRAME op."""
    frames = sorted({f for tick in TICKS for f, _, _ in tick if f != EMPTY})
    clouds = [synth.scan("vlp16_16k", frame=f, stride=8) for f in frames] + [np.zeros((0, 8), np.float32)]
    cloud_of = {f: i for i, f in enumerate(frames)}
    cloud_of[EMPTY] = len(frames)
    ops, kf_cloud, est = [], [], []
    for t, tick in enumerate(TICKS):
        first_new = len(kf_cloud)
        for f, acc, pf in tick:
            kf_cloud.append(cloud_of[f])
            est.append(synth.pose_matrix(pf) @ perturb(400 + len(est), 0.2, 1.0))  # graph estimates drift from the trajectory
            ops.append((KEYFRAME, cloud_of[f], acc, est[-1].copy()))
        ops.append((MAP, MAP_RES[t], [(k, est[k].copy()) for k in range(first_new)]))
        ops.append((DETECT,))
        for k in range(max(first_new, 1), len(kf_cloud)):  # odometry edges (:224-236): this keyframe's cloud on the previous one
            ops.append((INFO, 0, kf_cloud[k], kf_cloud[k - 1], np.linalg.inv(est[k - 1]) @ est[k]))
        ops.append((INFO, 1, kf_cloud[-1], kf_cloud[first_new], np.eye(4)))  # use_const_inf_matrix
        for k in range(len(est)):  # the optimiser moves every estimate
            est[k] = est[k] @ perturb(900 + 50 * t + k, 0.05, 0.3)
            ops.append((ESTIMATE, k, est[k].copy()))
    ops.append((MAP, MAP_RES[-1], [(k, est[k].copy()) for k in range(len(est))]))
    return clouds, ops


def write_input(path, params, clouds, ops):
    def iso(T):
        return np.ascontiguousarray(np.asarray(T, np.float64).T).tobytes()  # column-major
    with open(path, "wb") as f:
        f.write(struct.pack("<i", len(params)))
        for k, v in params.items():
            for s in (k.encode(), str(v).encode()):
                f.write(struct.pack("<i", len(s)) + s)
        f.write(struct.pack("<i", len(clouds)))
        for c in clouds:
            f.write(struct.pack("<i", c.shape[0]) + np.ascontiguousarray(c, np.float32).tobytes())
        f.write(struct.pack("<i", len(ops)))
        for op in ops:
            f.write(struct.pack("<i", op[0]))
            if op[0] == KEYFRAME:
                f.write(struct.pack("<id", op[1], op[2]) + iso(op[3]))
            elif op[0] == ESTIMATE:
                f.write(struct.pack("<i", op[1]) + iso(op[2]))
            elif op[0] == INFO:
                f.write(struct.pack("<iii", op[1], op[2], op[3]) + iso(op[4]))
            elif op[0] == MAP:
                f.write(struct.pack("<di", op[1], len(op[2])))
                for k, T in op[2]:
                    f.write(struct.pack("<i", k) + iso(T))


def read_blocks(path):
    data, blocks, i = open(path, "rb").read(), [], 0
    while i < len(data):
        n = struct.unpack_from("<q", data, i)[0]
        blocks.append(data[i + 8: i + 8 + n])
        i += 8 + n
    return blocks


def run_harness(harness, tmp_path, mode, params, clouds, ops):
    d = tmp_path / mode
    d.mkdir()
    write_input(d / "in.bin", params, clouds, ops)
    out = subprocess.run([harness, str(d), mode], capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout + out.stderr
    return read_blocks(d / "out.bin")


def parse_info(b, i=0):
    """a 6x6 information matrix as the harness writes it (rows, cols, column-major doubles) -> (matrix, next offset)"""
    r, c = struct.unpack_from("<ii", b, i)
    return np.frombuffer(b, np.float64, r * c, i + 8).reshape(c, r).T, i + 8 + 8 * r * c


def info_matrix(diag):
    inf = np.eye(6)
    inf[np.diag_indices(6)] = diag
    return inf


class Reference:
    """the reference's back end restated on one handle configured as the cache, and the oracle"""

    def __init__(self, params, clouds, oracle):
        self.clouds, self.oracle = clouds, oracle
        self.reg = pkg.select_registration_method({k: v for k, v in params.items() if k.startswith("reg") or k == "registration_method"})
        self.gate = pkg.LoopClosureGate(fitness_score_max_range=2.5)
        self.last = 0.0

    def detect(self, keyframes, new_keyframes):
        """loop_detector.hpp:57-171 on keyframes / new_keyframes = (accum, estimate, cloud index, keyframe index) -> the loops, the number
        of candidates, whether a new keyframe lost its candidates to a loop registered before it in this call, whether an empty cloud
        was a candidate"""
        loops, n_cands, gated, empty = [], 0, False, False
        planned = self.last
        for nk in new_keyframes:
            cands = ref_find_candidates(LOOP_PARAMS, [k[:2] for k in keyframes], nk[:2], self.last)
            gated |= not cands and bool(ref_find_candidates(LOOP_PARAMS, [k[:2] for k in keyframes], nk[:2], planned))
            n_cands += len(cands)
            best_score, best = DBL_MAX, None
            for c in cands:
                src, tgt = self.clouds[keyframes[c][2]], self.clouds[nk[2]]
                if src.shape[0] == 0 or tgt.shape[0] == 0:  # pcl::Registration::initCompute fails: hasConverged() is false
                    empty = True
                    continue
                self.reg.setInputTarget(tgt)
                self.reg.setInputSource(src)
                self.reg.align(self.gate.guess(nk[1], keyframes[c][1]))
                score = self.reg.getFitnessScore(2.5)
                if not self.reg.hasConverged() or score > best_score:  # :147
                    continue
                best_score, best = score, (keyframes[c][3], self.reg.getFinalTransformation())
            if best is not None and best_score <= 0.5:  # :160
                loops.append((nk[3], best[0], best[1]))
                self.last = nk[0]
        return loops, n_cands, gated, empty

    def information(self, c1, c2, relpose, const=False):
        if const:
            return info_matrix(pkg.information_from_fitness(0.0, use_const_inf_matrix=1))
        rel = np.asarray(relpose, np.float64).astype(np.float32)
        a, b = self.clouds[c1], self.clouds[c2]
        want, used, _ = self.oracle.fitness(a, b, rel, DBL_MAX)
        if used == 0:  # no neighbour in range (an empty cloud): calc_fitness_score returns DBL_MAX
            assert want == DBL_MAX
            score = DBL_MAX
        else:
            self.reg.setInputTarget(a)
            self.reg.setInputSource(b)
            score = self.reg.getFitnessScore(DBL_MAX, T=rel)
            assert abs(score - want) <= 1e-12 * want
        return info_matrix(pkg.information_from_fitness(score))

    def map(self, snaps, resolution):
        return self.reg.mapCloudGenerate([(self.clouds[c], T) for c, T in snaps], resolution)


@pytest.mark.parametrize("config", list(CONFIGS))
def test_backend_session(harness, synth, oracle, tmp_path, config):
    params = dict(CONFIGS[config], fitness_score_max_range="2.5")
    clouds, ops = session(synth)
    serial = run_harness(harness, tmp_path, "serial", params, clouds, ops)
    assert len(serial) == len(ops) + 1
    assert all(len(b) == 0 for op, b in zip(ops, serial) if op[0] in (KEYFRAME, ESTIMATE))
    ref = Reference(params, clouds, oracle)
    kf, registered, new, n_loops, n_cands, gated, empty_candidate = [], [], [], 0, [], False, False
    for op, b in zip(ops, serial):
        if op[0] == KEYFRAME:
            new.append([op[2], op[3], op[1], len(kf)])
            kf.append(new[-1])
        elif op[0] == ESTIMATE:
            kf[op[1]][1] = op[2]
        elif op[0] == DETECT:
            want, nc, g, e = ref.detect(registered, new)
            n_cands.append((len(registered), nc))
            gated, empty_candidate = gated or g, empty_candidate or e
            n, i = struct.unpack_from("<i", b)[0], 4
            got = []
            for _ in range(n):
                k1, k2 = struct.unpack_from("<ii", b, i)
                T = np.frombuffer(b, np.float32, 16, i + 8).reshape(4, 4).T
                inf, i = parse_info(b, i + 8 + 64)
                got.append((k1, k2, T, inf))
            last = struct.unpack_from("<d", b, i)[0]
            assert i + 8 == len(b)
            assert [(x[0], x[1]) for x in got] == [(w[0], w[1]) for w in want], (config, got, want)
            for x, w in zip(got, want):
                assert np.array_equal(x[2].view(np.uint32), w[2].view(np.uint32))  # relative_pose bitwise
                want_inf = ref.information(kf[x[0]][2], kf[x[1]][2], w[2].astype(np.float64))  # :569, relative_pose.cast<double>()
                assert np.array_equal(x[3].view(np.uint64), want_inf.view(np.uint64))
            assert last == ref.last  # last_edge_accum_distance after every tick
            n_loops += len(want)
            registered += new
            new = []
        elif op[0] == INFO:
            got, _ = parse_info(b)
            want = ref.information(op[2], op[3], op[4], const=op[1] == 1)
            assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (config, op[:4])
        elif op[0] == MAP:
            n = struct.unpack_from("<q", b)[0]
            want = ref.map([(kf[k][2], T) for k, T in op[2]], op[1])
            if not op[2]:
                assert n == -1 and want is None  # nullptr
                continue
            assert struct.unpack_from("<qqq", b, 8) == (n, 1, 0)  # width, height, is_dense
            assert len(b) == 32 + 32 * n
            assert b[32:] == np.ascontiguousarray(want, np.float32).tobytes(), (config, op[1])
    assert n_loops >= 3 and gated and empty_candidate
    assert n_cands[1][0] > 0 and n_cands[1][1] == 0  # the tick without candidates
    ref.reg.close()

    # one upload per keyframe cloud: the second pass on the same cache answers the same and uploads only pairs and poses
    h2d_first, h2d_again, n_first, n_again, same = struct.unpack("<QQqqq", serial[-1])
    assert same == 1
    assert n_first == n_again == len(clouds)
    assert h2d_first - h2d_again == sum(c.shape[0] for c in clouds) * 32

    # generate() on its own thread, detect() and the information matrices on this one: the serial answers
    concurrent = run_harness(harness, tmp_path, "concurrent", params, clouds, ops)
    assert concurrent[:-1] == serial[:-1]
