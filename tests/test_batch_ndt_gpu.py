"""GPU: NDT registrations in the device batch (b2r_batch_* on an NDT_OMP config, csrc/batch.cuh batch_run_ndt_chunk).  Every pair
runs the single handle's Newton / More-Thuente driver (NdtPairState) and its passes go through batched launches that reduce each
pair through its own chunk rows and fixed tree, so a pair's pose, flag, iteration count and fitness are BITWISE those of
b2r_set_target / b2r_set_source / b2r_align / b2r_fitness on one NDT handle, whatever else shares the batch.
Reference site: LoopDetector::matching (include/hdl_graph_slam/loop_detector.hpp:117-171) with the factory's default NDT_OMP."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg
from common import rot_err, trans_err, perturb

pytestmark = pytest.mark.gpu

MAXR = 2.5


def ndt_cfg(res=1.0, search=7, flag=0, fixed=0, max_iterations=64):
    c = pkg.default_config(pkg.B2R_METHOD_NDT)
    c.ndt_resolution = res
    c.ndt_search_method = search
    c.ndt_mt_interval_flag = flag
    c.ndt_fixed_iterations = fixed
    c.max_iterations = max_iterations
    return c


def groups(synth, sensor="vlp16_16k", targets=(0, 10), cands=(1, 251, 2, 252), seed=60):
    clouds, pairs = {}, []
    for gi, tf in enumerate(targets):
        clouds.setdefault(tf, synth.scan(sensor, frame=tf, stride=8))
        for j, off in enumerate(cands):
            sf = tf + off
            clouds.setdefault(sf, synth.scan(sensor, frame=sf, stride=8))
            rel = np.linalg.inv(synth.pose_matrix(tf)) @ synth.pose_matrix(sf)
            g = (rel @ perturb(seed + 7 * gi + j, 0.3, 2.0)).astype(np.float32)
            g[2, 3] = 0.0
            pairs.append((sf, tf, g))
    return clouds, pairs


def run_batch(cfg, clouds, pairs, want_fitness=True):
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {k: lb.addCloud(c) for k, c in clouds.items()}
    res = lb.align([(ids[s], ids[t], g) for s, t, g in pairs], want_fitness, MAXR)
    rounds = lb.lastRounds()
    lb.close()
    return res, rounds


def run_single(cfg, clouds, pairs):
    r = pkg.Registration(cfg)
    out = []
    for s, t, g in pairs:
        r.setInputTarget(clouds[t])
        r.setInputSource(clouds[s])
        r.align(g)
        out.append({"T": r.getFinalTransformation(), "converged": r.hasConverged(), "iterations": r.nr_iterations,
                    "fitness": r.getFitnessScore(MAXR)})
    r.close()
    return out


def same(a, b, fitness=True):
    ok = np.array_equal(np.asarray(a["T"]).view(np.uint32), np.asarray(b["T"]).view(np.uint32))
    ok = ok and bool(a["converged"]) == bool(b["converged"]) and a["iterations"] == b["iterations"]
    if fitness:
        ok = ok and np.float64(a["fitness"]).tobytes() == np.float64(b["fitness"]).tobytes()
    return ok


@pytest.mark.parametrize("res,search,flag,fixed", [(1.0, 7, 0, 0), (0.5, 7, 0, 0), (1.0, 1, 0, 0), (0.5, 1, 0, 0), (1.0, 7, 1, 0), (1.0, 7, 0, 6)])
def test_batch_equals_single_handle(synth, res, search, flag, fixed):
    cfg = ndt_cfg(res, search, flag, fixed)
    clouds, pairs = groups(synth)
    got, (rounds, pair_rounds) = run_batch(cfg, clouds, pairs)
    want = run_single(cfg, clouds, pairs)
    for i, (a, b) in enumerate(zip(got, want)):
        assert same(a, b), f"pair {i}"
    assert rounds >= 2 and pair_rounds >= rounds
    if fixed:
        assert all(r["iterations"] == fixed for r in got)
    nofit, _ = run_batch(cfg, clouds, pairs, want_fitness=False)
    for a, b in zip(nofit, got):
        assert same(a, b, fitness=False) and np.isnan(a["fitness"])


def test_mixed_sizes_shared_targets_and_early_and_capped_pairs(synth):
    """targets shared by groups of 8 sources of 16 384 / 65 536 / 131 072 / 262 144 points; a low iteration cap so that some pairs
    stop at it while others (a source that IS its target) converge early, and pairs of different pass kinds share rounds"""
    sizes = ["vlp16_16k", "vlp16", "hdl32e", (64, 4096)]
    clouds, pairs = {}, []
    for gi, tf in enumerate((0, 40)):
        clouds[("t", tf)] = synth.scan(sizes[gi], frame=tf, stride=8)
        for j in range(8):
            sf = tf + 1 + j
            key = ("s", sf, j % 4)
            clouds[key] = synth.scan(sizes[j % 4], frame=sf, stride=8)
            rel = np.linalg.inv(synth.pose_matrix(tf)) @ synth.pose_matrix(sf)
            pairs.append((key, ("t", tf), (rel @ perturb(90 + 8 * gi + j, 0.4, 3.0)).astype(np.float32)))
        pairs.append((("t", tf), ("t", tf), np.eye(4, dtype=np.float32)))
    for flag in (0, 1):
        cfg = ndt_cfg(1.0, 7, flag, 0, max_iterations=3)
        got, _ = run_batch(cfg, clouds, pairs)
        want = run_single(cfg, clouds, pairs)
        for i, (a, b) in enumerate(zip(got, want)):
            assert same(a, b), f"flag {flag} pair {i}"
        its = [r["iterations"] for r in got]
        assert min(its) < max(its)


def test_degenerate_pairs(synth):
    tgt = synth.scan("vlp16_16k", frame=0, stride=8)
    src = synth.scan("vlp16_16k", frame=1, stride=8)
    nan_src = src.copy()
    nan_src[::7, :3] = np.nan
    nan_src[3::11, 1] = np.inf
    sparse = tgt[:4].copy()  # geometry exists, but no voxel has 6 points
    all_nan = np.full((64, 8), np.nan, np.float32)
    empty = np.zeros((0, 8), np.float32)
    clouds = {"t": tgt, "s": src, "nan": nan_src, "sparse": sparse, "allnan": all_nan, "empty": empty}
    G = perturb(5, 0.2, 1.0).astype(np.float32)
    pairs = [("s", "t", G), ("empty", "t", G), ("s", "empty", G), ("s", "sparse", G), ("s", "allnan", G), ("nan", "t", G), ("s", "t", np.eye(4, dtype=np.float32))]
    cfg = ndt_cfg(1.0)
    got, _ = run_batch(cfg, clouds, pairs)
    want = run_single(cfg, clouds, pairs)
    for i, (a, b) in enumerate(zip(got, want)):
        assert same(a, b), f"pair {i}"
    assert got[1]["fitness"] == np.finfo(np.float64).max and not got[1]["converged"]


def test_co_scheduled_pairs_do_not_matter(synth):
    clouds, pairs = groups(synth, targets=tuple(range(0, 250, 10)), cands=(1, 2, 3, 251, 252, 253, 4, 254))
    assert len(pairs) == 200
    cfg = ndt_cfg(1.0)
    lb = pkg.RegistrationBatch(cfg=cfg)
    ids = {k: lb.addCloud(c) for k, c in clouds.items()}
    pl = [(ids[s], ids[t], g) for s, t, g in pairs]
    full = lb.align(pl, True, MAXR)
    again = lb.align(pl, True, MAXR)
    rev = lb.align(pl[::-1], True, MAXR)[::-1]
    for i in range(200):
        assert same(full[i], again[i]) and same(full[i], rev[i]), f"pair {i}"
    for i in (0, 77, 199):
        assert same(lb.align([pl[i]], True, MAXR)[0], full[i])
    lb.close()
    want = run_single(cfg, clouds, [pairs[i] for i in (0, 100, 199)])
    for i, w in zip((0, 100, 199), want):
        assert same(full[i], w)


@pytest.mark.parametrize("case", [0, 1, 2, 3])
def test_batch_matches_oracle(synth, oracle, case):
    src, tgt = synth.scan("vlp16_16k", frame=1, stride=8), synth.scan("vlp16_16k", frame=0, stride=8)
    res, search, guess = [(1.0, 7, None), (1.0, 7, 11), (0.5, 1, 12), (1.0, 1, 13)][case]
    G = (np.eye(4) if guess is None else perturb(guess, 0.3, 1.5)).astype(np.float32)
    got, _ = run_batch(ndt_cfg(res, search), {"s": src, "t": tgt}, [("s", "t", G), ("t", "t", G)])
    o = oracle.NdtMap(tgt, res).align(src, G, search_method=search)
    assert bool(got[0]["converged"]) == o["converged"] and got[0]["iterations"] == o["iterations"]
    assert trans_err(got[0]["T"], o["T"]) < 1e-4 and rot_err(got[0]["T"], o["T"]) < 1e-4


def test_loop_matching_on_ndt_handle_equals_sequential_calls(synth):
    clouds, pairs = groups(synth, targets=(0,), cands=(1, 251, 2, 252, 3))
    reg = pkg.select_registration_method({"registration_method": "NDT_OMP", "reg_resolution": 1.0})
    det = pkg.LoopDetector(reg, fitness_score_max_range=MAXR, fitness_score_thresh=0.5)
    best, rs = det.matching([clouds[s] for s, _, _ in pairs], clouds[0], [g for _, _, g in pairs])
    cfg = reg.config
    reg.close()
    want = run_single(cfg, clouds, pairs)
    for a, b in zip(rs, want):
        assert same(a, b)
    assert best == pkg.loop_argmin([_as_result(q) for q in want], 0.5)


def _as_result(d):
    from hdl_graph_slam_b200 import _capi
    r = _capi.Result()
    r.fitness, r.converged, r.iterations = d["fitness"], int(d["converged"]), d["iterations"]
    return r


def test_loop_detect_single_rank_equals_align_plus_argmin(synth):
    clouds, pairs = groups(synth, targets=(0, 10), cands=(1, 251, 2))
    group_first = [0, 3, 6]
    lb = pkg.RegistrationBatch(cfg=ndt_cfg(1.0))
    ids = {f: lb.addCloud(c) for f, c in clouds.items()}
    pl = [(ids[s], ids[t], g) for s, t, g in pairs]
    res = lb.align(pl, True, MAXR)
    best, allres = lb.loopDetect(pl, group_first, MAXR, 0.5)
    for a, b in zip(res, allres):
        assert same(a, b)
    for g in range(2):
        assert best[g] == pkg.loop_argmin([_as_result(q) for q in res[group_first[g]: group_first[g + 1]]], 0.5)
    lb.close()


def test_detect_plan_batch_replay_equals_the_sequential_walk(synth):
    from test_loop_gate import ref_find_candidates
    kf_frames = [0, 2, 10, 12, 20, 120]
    new_frames = [251, 253, 261, 271]
    kfs = [(float(f), synth.pose_matrix(f)) for f in kf_frames]
    news = [(float(f), synth.pose_matrix(f) @ perturb(300 + f, 0.2, 1.0)) for f in new_frames]
    clouds = {f: synth.scan("vlp16_16k", frame=f, stride=8) for f in kf_frames + new_frames}
    p = dict(distance_thresh=5.0, accum_distance_thresh=8.0, min_edge_interval=5.0)
    gate = pkg.LoopClosureGate(fitness_score_max_range=MAXR)
    params = {"registration_method": "NDT_OMP", "reg_resolution": 1.0}
    reg = pkg.select_registration_method(params)
    det = pkg.LoopDetector(reg, fitness_score_max_range=MAXR, fitness_score_thresh=0.5)
    last, want = 0.0, []
    for gi, nk in enumerate(news):
        cands = ref_find_candidates(p, kfs, nk, last)
        if not cands:
            continue
        guesses = [gate.guess(nk[1], kfs[c][1]) for c in cands]
        # the reference's walk: one setInputSource / align / getFitnessScore per candidate on one handle
        rs = run_single(reg.config, {**{("k", c): clouds[kf_frames[c]] for c in cands}, "n": clouds[new_frames[gi]]},
                        [(("k", c), "n", g) for c, g in zip(cands, guesses)])
        best = pkg.loop_argmin([_as_result(q) for q in rs], 0.5)
        if best >= 0:
            want.append((gi, cands[best], rs[best]["T"]))
            last = nk[0]
    cfg = reg.config
    reg.close()
    assert len(want) >= 1
    lb = pkg.RegistrationBatch(cfg=cfg)
    kid = [lb.addCloud(clouds[f]) for f in kf_frames]
    nid = [lb.addCloud(clouds[f]) for f in new_frames]
    got = gate.detect(lb, kfs, kid, news, nid)
    lb.close()
    assert [(g, c) for g, c, _ in got] == [(g, c) for g, c, _ in want]
    for (_, _, Ta), (_, _, Tb) in zip(got, want):
        assert np.array_equal(Ta, Tb)


def test_fitness_and_map_cloud_on_ndt_batch_equal_gicp_batch(synth):
    frames = {f: synth.scan("vlp16_16k", frame=f, stride=8) for f in (0, 1, 2, 30)}
    edges = [(a, b_, (np.linalg.inv(synth.pose_matrix(a)) @ synth.pose_matrix(b_)).astype(np.float32)) for a, b_ in ((0, 1), (1, 2), (0, 30))]
    poses = [synth.pose_matrix(f).astype(np.float32) for f in frames]
    out = []
    for cfg in (ndt_cfg(1.0), pkg.default_config(pkg.B2R_METHOD_GICP)):
        lb = pkg.RegistrationBatch(cfg=cfg)
        ids = {f: lb.addCloud(c) for f, c in frames.items()}
        sc = lb.calcFitnessScore([(ids[a], ids[b_], rel) for a, b_, rel in edges], 2.0)
        m1 = lb.mapCloudGenerate([ids[f] for f in frames], poses, 0.5)
        m0 = lb.mapCloudGenerate([ids[f] for f in frames], poses, 0.0)
        out.append((sc, m1, m0))
        lb.close()
    (sa, ma1, ma0), (sb, mb1, mb0) = out
    assert sa.tobytes() == sb.tobytes()
    assert np.array_equal(ma1, mb1) and np.array_equal(ma0, mb0)
