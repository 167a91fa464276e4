"""GPU: the back-end drop-in (adapter/b200_backend.hpp, through tests/backend_harness.cpp) over the session of
test_backend_adapter_gpu.py on every registration branch the factory serves beyond FastGICP and NDT_OMP: pcl GICP, pclomp GICP, pcl ICP
with reciprocal correspondences off and on, FastVGICP, FastVGICPCuda, pcl NDT, NDT_OMP's KDTREE search and NDT_OMP with DIRECT1.

For each method:
  - the loops and last_edge_accum_distance after every tick are the reference walk's on one handle, relative poses bitwise; the
    session registers at least one loop and turns down at least one new keyframe whose best candidate fails fitness_score_thresh;
  - every registered loop's align, re-run by the method's own sequential reference (tests/method_refs.py) from the same guess, gives the
    same iterations and flag and the pose within that method's tolerance;
  - the empty keyframe cloud: as a loop candidate its batch record is a fresh single handle's, and as cloud1 of an information edge it
    gives DBL_MAX and the information of that score;
  - information matrices bitwise b2r_information_from_fitness(b2r_fitness) on a fresh handle and within 1e-12 of the oracle's
    calc_fitness_score; maps bitwise b2r_map_cloud_generate at 0.05, 0 and -1; one upload per keyframe cloud.
Under every reg_* key a branch reads set away from its default, the session is bitwise the raw ABI's with that dict and differs from the
default set's."""
import struct

import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from method_refs import METHODS, NON_DEFAULT, References, pose_close
from test_backend_adapter_gpu import DBL_MAX, DETECT, ESTIMATE, INFO, KEYFRAME, LOOP_PARAMS, MAP, Reference, harness, parse_info, run_harness, session  # noqa: F401
from test_loop_gate import ref_find_candidates

pytestmark = pytest.mark.gpu
CASES = ["GICP", "B200_GICP_OMP", "B200_ICP", "B200_ICP_reciprocal", "FAST_VGICP", "B200_VGICP_CUDA", "NDT", "B200_NDT_KDTREE",
         "NDT_OMP_DIRECT1"]
FITNESS_THRESH = 0.5  # LoopDetector's default fitness_score_thresh


@pytest.fixture(scope="module")
def refs(tmp_path_factory, oracle):
    r = References(tmp_path_factory, oracle)
    yield r
    r.close()


class MethodReference(Reference):
    """Reference's walk (loop_detector.hpp:57-171 on one handle), also recording every registered loop's align, the new keyframes whose
    best converged candidate failed fitness_score_thresh, and the empty-cloud candidates"""

    def __init__(self, params, clouds, oracle):
        super().__init__(params, clouds, oracle)
        self.thresh = float(params.get("fitness_score_thresh", FITNESS_THRESH))
        self.loop_aligns, self.loop_scores, self.over_thresh, self.empty_pairs = [], [], 0, []

    def information(self, c1, c2, relpose, const=False):
        """InformationMatrixCalculator reads the same fitness_score_thresh rosparam as LoopDetector (information_matrix_calculator.cpp)"""
        got = super().information(c1, c2, relpose, const)
        if const or self.thresh == FITNESS_THRESH:
            return got
        rel = np.asarray(relpose, np.float64).astype(np.float32)
        score = self.oracle.fitness(self.clouds[c1], self.clouds[c2], rel, DBL_MAX)[0] if self.clouds[c1].shape[0] else DBL_MAX
        if score != DBL_MAX:
            self.reg.setInputTarget(self.clouds[c1])
            self.reg.setInputSource(self.clouds[c2])
            score = self.reg.getFitnessScore(DBL_MAX, T=rel)
        return np.diag(pkg.information_from_fitness(score, fitness_score_thresh=self.thresh))

    def detect(self, keyframes, new_keyframes):
        loops, n_cands, gated, empty = [], 0, False, False
        planned = self.last
        for nk in new_keyframes:
            cands = ref_find_candidates(LOOP_PARAMS, [k[:2] for k in keyframes], nk[:2], self.last)
            gated |= not cands and bool(ref_find_candidates(LOOP_PARAMS, [k[:2] for k in keyframes], nk[:2], planned))
            n_cands += len(cands)
            best_score, best = DBL_MAX, None
            for c in cands:
                src, tgt = self.clouds[keyframes[c][2]], self.clouds[nk[2]]
                guess = self.gate.guess(nk[1], keyframes[c][1])
                if src.shape[0] == 0 or tgt.shape[0] == 0:
                    empty = True
                    self.empty_pairs.append((keyframes[c][2], nk[2], guess))
                    continue
                self.reg.setInputTarget(tgt)
                self.reg.setInputSource(src)
                self.reg.align(guess)
                score = self.reg.getFitnessScore(2.5)
                if not self.reg.hasConverged() or score > best_score:
                    continue
                best_score = score
                best = (keyframes[c][3], self.reg.getFinalTransformation(), keyframes[c][2], nk[2], guess, self.reg.nr_iterations)
            if best is not None and best_score <= self.thresh:
                loops.append((nk[3], best[0], best[1]))
                self.loop_aligns.append(best[1:])
                self.loop_scores.append(best_score)
                self.last = nk[0]
            elif best is not None:
                self.over_thresh += 1
        return loops, n_cands, gated, empty


def replay_session(harness, tmp_path, params, clouds, ops, oracle, gate=True):
    """the session through the drop-in against MethodReference, every answer checked -> (the reference, the harness blocks)"""
    serial = run_harness(harness, tmp_path, "serial", params, clouds, ops)
    assert len(serial) == len(ops) + 1
    ref = MethodReference(params, clouds, oracle)
    kf, registered, new, n_loops, empty_cloud1, gated, n_cands = [], [], [], 0, False, False, []
    for op, b in zip(ops, serial):
        if op[0] == KEYFRAME:
            new.append([op[2], op[3], op[1], len(kf)])
            kf.append(new[-1])
        elif op[0] == ESTIMATE:
            kf[op[1]][1] = op[2]
        elif op[0] == DETECT:
            want, nc, g, _ = ref.detect(registered, new)
            n_cands.append((len(registered), nc))
            gated = gated or g
            n, i = struct.unpack_from("<i", b)[0], 4
            got = []
            for _ in range(n):
                k1, k2 = struct.unpack_from("<ii", b, i)
                T = np.frombuffer(b, np.float32, 16, i + 8).reshape(4, 4).T
                inf, i = parse_info(b, i + 8 + 64)
                got.append((k1, k2, T, inf))
            assert struct.unpack_from("<d", b, i)[0] == ref.last and i + 8 == len(b)
            assert [(x[0], x[1]) for x in got] == [(w[0], w[1]) for w in want], (got, want)
            for x, w in zip(got, want):
                assert np.array_equal(x[2].view(np.uint32), w[2].view(np.uint32))
                want_inf = ref.information(kf[x[0]][2], kf[x[1]][2], w[2].astype(np.float64))
                assert np.array_equal(x[3].view(np.uint64), want_inf.view(np.uint64))
            n_loops += len(want)
            registered += new
            new = []
        elif op[0] == INFO:
            got, _ = parse_info(b)
            want = ref.information(op[2], op[3], op[4], const=op[1] == 1)
            assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), op[:4]
            if op[1] == 0 and clouds[op[2]].shape[0] == 0:  # cloud1 empty: no neighbour, calc_fitness_score's DBL_MAX
                empty_cloud1 = True
                assert np.array_equal(got, np.diag(np.diag(got)))
                assert np.array_equal(got.view(np.uint64), np.diag(pkg.information_from_fitness(DBL_MAX, fitness_score_thresh=ref.thresh)).view(np.uint64))
        elif op[0] == MAP:
            n = struct.unpack_from("<q", b)[0]
            want = ref.map([(kf[k][2], T) for k, T in op[2]], op[1])
            if not op[2]:
                assert n == -1 and want is None
                continue
            assert struct.unpack_from("<qqq", b, 8) == (n, 1, 0) and len(b) == 32 + 32 * n
            assert b[32:] == np.ascontiguousarray(want, np.float32).tobytes(), op[1]
    assert empty_cloud1 and ref.empty_pairs
    assert gated or not gate  # a keyframe whose candidates a loop registered earlier in the same tick gates out
    assert n_cands[1][0] > 0 and n_cands[1][1] == 0  # the tick without candidates
    h2d_first, h2d_again, n_first, n_again, same = struct.unpack("<QQqqq", serial[-1])
    assert same == 1 and n_first == n_again == len(clouds)
    assert h2d_first - h2d_again == sum(c.shape[0] for c in clouds) * 32
    ref.n_loops = n_loops
    return ref, serial


@pytest.mark.parametrize("case", CASES)
def test_backend_session_on_every_method(harness, synth, oracle, refs, tmp_path, case):
    reg = METHODS[case]
    clouds, ops = session(synth)
    # At the default fitness_score_thresh = 0.5 every method registers every loop the session offers.  So that the threshold is
    # exercised too, the session runs again with the threshold midway between the two best scores of those loops: the walk must then
    # turn down at least one new keyframe for its fitness and still register one
    for d in ("default", "between"):
        (tmp_path / d).mkdir()
    params = dict(reg, fitness_score_max_range="2.5", fitness_score_thresh=str(FITNESS_THRESH))
    ref, _ = replay_session(harness, tmp_path / "default", params, clouds, ops, oracle)
    assert ref.n_loops >= 2, (case, ref.n_loops)
    ref.reg.close()
    lo, hi = sorted(ref.loop_scores)[:2]
    assert hi > lo
    params["fitness_score_thresh"] = repr(0.5 * (lo + hi))
    # (the raised threshold may turn down the loop that gates a later keyframe of its tick: the first pass took the gate)
    ref, _ = replay_session(harness, tmp_path / "between", params, clouds, ops, oracle, gate=False)
    assert ref.n_loops >= 1 and ref.over_thresh >= 1, (case, ref.n_loops, ref.over_thresh)
    cfg = ref.reg.config

    # every registered loop against the method's own sequential reference, from the same guess
    for T, s, t, guess, iterations in ref.loop_aligns:
        w = refs.align(case, cfg, clouds[s], clouds[t], guess)
        assert w["converged"] and w["iterations"] == iterations, (case, s, t, w["iterations"], iterations)
        assert pose_close(case, T, w["T"]), (case, s, t, np.max(np.abs(T - w["T"])))

    # the empty keyframe as a loop candidate: in one group with a registered loop's candidate (same target, same guess), its batch
    # record is a fresh single handle's, fitness included, and the loop's candidate still wins the group
    s, _, _ = ref.empty_pairs[0]
    _, ls, lt, lguess, _ = ref.loop_aligns[0]
    b = pkg.RegistrationBatch(params=reg)
    ids = [b.addCloud(c) for c in clouds]
    best, recs = b.loopDetect([(ids[s], ids[lt], lguess), (ids[ls], ids[lt], lguess)], [0, 2], 2.5, ref.thresh)
    b.close()
    single = pkg.select_registration_method(reg)
    single.setInputTarget(clouds[lt])
    single.setInputSource(clouds[s])
    single.align(lguess)
    e = recs[0]
    assert (e["converged"], e["iterations"]) == (single.hasConverged(), single.nr_iterations) == (False, 0), (case, e)
    assert e["T"].view(np.uint32).tobytes() == single.getFinalTransformation().view(np.uint32).tobytes()
    assert np.float64(e["fitness"]).tobytes() == np.float64(single.getFitnessScore(2.5)).tobytes(), (e["fitness"], single.getFitnessScore(2.5))
    assert best == [1], best
    single.close()
    ref.reg.close()


@pytest.mark.parametrize("branch", list(NON_DEFAULT))
def test_non_default_session_is_the_raw_session(harness, synth, oracle, tmp_path, branch):
    """every reg_* key the branch reads, away from its default: the drop-in's session is bitwise the raw ABI's with that dict, and is
    not the default set's session"""
    clouds, ops = session(synth)
    extra = dict(fitness_score_max_range="2.5", fitness_score_thresh=str(FITNESS_THRESH))
    for d in ("set", "default"):
        (tmp_path / d).mkdir()
    ref, blocks = replay_session(harness, tmp_path / "set", dict(NON_DEFAULT[branch], **extra), clouds, ops, oracle)
    ref.reg.close()
    default = run_harness(harness, tmp_path / "default", "serial", dict(registration_method=NON_DEFAULT[branch]["registration_method"], **extra),
                          clouds, ops)
    assert blocks[:-1] != default[:-1]
