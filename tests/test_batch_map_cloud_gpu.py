"""GPU: MapCloudGenerator::generate (src/hdl_graph_slam/map_cloud_generator.cpp:13-51) over the keyframe clouds a b2r_batch
already caches (b2r_batch_map_cloud_generate).

- bitwise equal, row for row, to b2r_map_cloud_generate on the same clouds and poses, at three resolutions and unfiltered, with
  NaN / +-inf points, empty keyframes first, in between and last, ids out of order and one id repeated;
- the same SET of voxel centres as the oracle's octree;
- device-added clouds: read through their search structure once it is built (also when the map call builds it), refused where the
  full records are needed (resolution <= 0), as is a record stride other than the output's;
- mixed 16- and 32-byte cloud records; no point upload; align / loop detection / fitness scores unchanged by map calls in between;
- map scale: 250 keyframes, about 4.1 M points, and the octree-depth limit."""
import numpy as np
import pytest
import torch  # before the engine library: it links the system NCCL, and torch's CUDA libraries must resolve against their own first
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import _capi
from common import perturb

pytestmark = pytest.mark.gpu

GICP = {"registration_method": "FAST_GICP"}
EMPTY = np.zeros((0, 8), np.float32)


def decorate(cloud, seed):
    """a copy with exact lattice ties (every 97th point rounded to whole metres) and a few NaN / +-inf points"""
    c = np.array(cloud, np.float32, copy=True)
    c[::97, :3] = np.round(c[::97, :3])
    bad = np.random.default_rng(seed).choice(c.shape[0], 6, replace=False)
    c[bad[0], 0] = np.nan
    c[bad[1], 1] = np.nan
    c[bad[2], 2] = np.inf
    c[bad[3], 0] = -np.inf
    c[bad[4], :3] = np.nan
    c[bad[5], 1] = np.inf
    return c


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def same_rows(got, want):
    assert got.shape == want.shape
    assert np.array_equal(bits(got), bits(want))


def to_device(cloud):
    d = torch.from_numpy(np.ascontiguousarray(cloud)).cuda()
    torch.cuda.synchronize()
    return d


def from_device(ptr, m, stride_f):
    """copy m records at an engine-owned device pointer to the host"""
    from cuda.bindings import runtime as cudart
    copy = torch.empty((m, stride_f), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    if m:
        err, = cudart.cudaMemcpy(copy.data_ptr(), ptr, m * stride_f * 4, cudart.cudaMemcpyKind.cudaMemcpyDeviceToDevice)
        assert int(err) == 0
    return copy.cpu().numpy()


@pytest.fixture(scope="module")
def scene(synth):
    """clouds (added in this order) and a keyframe list over them: empty keyframes first, in between and last, the clouds out of
    their add order, cloud 3 named twice at two poses"""
    frames = (0, 5, 10, 60, 130)
    clouds = [EMPTY] + [decorate(synth.scan("vlp16_16k", frame=f, stride=8), seed=f) for f in frames[:3]] + [EMPTY]
    clouds += [decorate(synth.scan("vlp16_16k", frame=f, stride=8), seed=f) for f in frames[3:]] + [EMPTY]
    frame_of = {1: 0, 2: 5, 3: 10, 5: 60, 6: 130}
    pose = lambda i, s: synth.pose_matrix(frame_of.get(i, 0)) @ perturb(s, 0.05, 0.5)  # noqa: E731
    order = [0, 3, 1, 4, 2, 6, 3, 5, 7]
    poses = [pose(i, k) for k, i in enumerate(order)]
    return clouds, order, poses


def host_map(lb, clouds, order, poses, res):
    return lb.engine.mapCloudGenerate([(clouds[i], P) for i, P in zip(order, poses)], res)


@pytest.mark.parametrize("res", [0.05, 0.25, 1.0, 0.0])
def test_equals_host_entry_point_row_for_row(scene, res):
    clouds, order, poses = scene
    lb = pkg.RegistrationBatch(params=GICP)
    ids = [lb.addCloud(c) for c in clouds]
    got = lb.mapCloudGenerate([ids[i] for i in order], poses, res)
    want = host_map(lb, clouds, order, poses, res)
    assert want.shape[0] > 0
    same_rows(got, want)
    # the device result is the same records, and a second call repeats them bitwise
    ptr, m = lb.mapCloudGenerate([ids[i] for i in order], poses, res, device=True)
    same_rows(from_device(ptr, m, 8), want)
    assert lb.mapCloudGenerate([], [], res) is None  # "warning: keyframes empty!!"
    lb.close()


@pytest.mark.parametrize("res", [0.05, 0.25, 1.0])
def test_voxel_centres_equal_the_oracle_octree(scene, oracle, res):
    clouds, order, poses = scene
    lb = pkg.RegistrationBatch(params=GICP)
    ids = [lb.addCloud(c) for c in clouds]
    got = lb.mapCloudGenerate([ids[i] for i in order], poses, res)
    want = oracle.map_cloud_generate([(clouds[i], P) for i, P in zip(order, poses)], res)
    assert got.shape[0] == want.shape[0] > 0
    g = got[:, :3]
    g = g[np.lexsort((g[:, 0], g[:, 1], g[:, 2]))]
    assert np.array_equal(g, want)
    assert np.all(got[:, 3] == 1.0) and np.all(got[:, 4:] == 0.0)
    lb.close()


def test_device_added_clouds_are_read_through_their_structures(scene):
    clouds, order, poses = scene
    keep = [k for k, i in enumerate(order) if clouds[i].shape[0]]
    order, poses = [order[k] for k in keep], [poses[k] for k in keep]
    lb = pkg.RegistrationBatch(params=GICP)
    host = {i: lb.addCloud(clouds[i]) for i in set(order)}
    want = lb.mapCloudGenerate([host[i] for i in order], poses, 0.25)
    same_rows(want, host_map(lb, clouds, order, poses, 0.25))
    # aligned once, then the caller's buffers are overwritten: the map comes from the structures
    dev = {i: to_device(clouds[i]) for i in set(order)}
    ids = {i: lb.addCloudRaw(d.data_ptr(), d.shape[0], d.shape[1] * 4, device=True) for i, d in dev.items()}
    lb.align([(ids[1], ids[2], np.eye(4)), (ids[5], ids[6], np.eye(4)), (ids[3], ids[1], np.eye(4))])
    for d in dev.values():
        d.fill_(7.0)
    torch.cuda.synchronize()
    same_rows(lb.mapCloudGenerate([ids[i] for i in order], poses, 0.25), want)
    # never aligned: the map call builds the structures (the buffers are live until then), and they serve every later call
    fresh = {i: to_device(clouds[i]) for i in set(order)}
    ids2 = {i: lb.addCloudRaw(d.data_ptr(), d.shape[0], d.shape[1] * 4, device=True) for i, d in fresh.items()}
    same_rows(lb.mapCloudGenerate([ids2[i] for i in order], poses, 0.25), want)
    for d in fresh.values():
        d.fill_(-3.0)
    torch.cuda.synchronize()
    same_rows(lb.mapCloudGenerate([ids2[i] for i in order], poses, 0.25), want)
    lb.close()


def test_unfiltered_map_needs_records_the_batch_holds(scene, synth):
    clouds, _, _ = scene
    lb = pkg.RegistrationBatch(params=GICP)
    a = lb.addCloud(clouds[1])
    d = to_device(clouds[2])
    dv = lb.addCloudRaw(d.data_ptr(), d.shape[0], 32, device=True)
    c16 = np.ascontiguousarray(synth.scan("vlp16_16k", frame=3, stride=4))
    s16 = lb.addCloud(c16)
    I = np.eye(4)
    with pytest.raises(pkg.B2RError) as e:
        lb.mapCloudGenerate([a, dv], [I, I], 0.0)
    assert e.value.code == _capi.B2R_EINVAL and f"cloud id {dv} " in str(e.value) and "device memory" in str(e.value)
    with pytest.raises(pkg.B2RError) as e:
        lb.mapCloudGenerate([a, s16], [I, I], 0.0)
    assert e.value.code == _capi.B2R_EINVAL and f"cloud id {s16} " in str(e.value) and "16-byte" in str(e.value)
    # the batch still works: the same clouds at a resolution, the 16-byte cloud unfiltered at its own stride, an align
    assert lb.mapCloudGenerate([a, dv, s16], [I, I, I], 0.25).shape[0] > 0
    same_rows(lb.mapCloudGenerate([s16], [I], 0.0, stride_bytes=16), lb.engine.mapCloudGenerate([(c16, I)], 0.0))
    assert len(lb.align([(a, dv, I)])) == 1
    lb.close()


@pytest.mark.parametrize("res", [0.05, 0.25])
def test_mixed_record_strides(scene, synth, res):
    clouds, order, poses = scene
    lb = pkg.RegistrationBatch(params=GICP)
    ids, as32 = [], []
    for k, c in enumerate(clouds):
        if k % 2:  # every other cloud as 16-byte x y z 1 records
            c16 = np.ascontiguousarray(c[:, :4])
            ids.append(lb.addCloud(c16))
            pad = np.zeros((c.shape[0], 8), np.float32)
            pad[:, :4] = c16
            as32.append(pad)
        else:
            ids.append(lb.addCloud(c))
            as32.append(c)
    got = lb.mapCloudGenerate([ids[i] for i in order], poses, res)
    same_rows(got, host_map(lb, as32, order, poses, res))
    lb.close()


def test_no_point_upload(scene):
    clouds, order, poses = scene
    lb = pkg.RegistrationBatch(params=GICP)
    ids = [lb.addCloud(c) for c in clouds]
    kf = [ids[i] for i in order]
    lb.align([(ids[1], ids[2], np.eye(4))])  # some structures built, others not: the map call builds those
    lb.synchronize()
    for res in (0.25, 0.0):
        h0 = lb.engine.getStats()["h2d_bytes"]
        lb.mapCloudGenerate(kf, poses, res)
        h1 = lb.engine.getStats()["h2d_bytes"]
        assert h1 - h0 <= len(kf) * 64
        host_map(lb, clouds, order, poses, res)
        h2 = lb.engine.getStats()["h2d_bytes"]
        assert h2 - h1 == sum(clouds[i].shape[0] for i in order) * 32
    lb.close()


def _results_bits(res):
    return [(bytes(r.T), r.fitness, r.converged, r.iterations) for r in res]


def test_map_calls_do_not_disturb_the_batch(synth, scene):
    clouds, order, poses = scene
    frames = {f: synth.scan("vlp16_16k", frame=f, stride=8) for f in (0, 1, 2, 3)}
    g = [perturb(k, 0.2, 1.0) for k in range(4)]
    pairs = [(1, 0, g[0]), (2, 0, g[1]), (3, 0, g[2]), (2, 1, g[3]), (3, 1, np.eye(4))]

    def run(with_map):
        lb = pkg.RegistrationBatch(params=GICP)
        ids = {f: lb.addCloud(c) for f, c in frames.items()}
        extra = [lb.addCloud(c) for c in clouds]
        pl = [(ids[s], ids[t], G) for s, t, G in pairs]
        all_ids = [ids[f] for f in frames] + extra
        I = [np.eye(4)] * len(all_ids)
        maps = []
        if with_map:  # structures built by the map call, covariances by the align after it
            maps.append(lb.mapCloudGenerate(all_ids, I, 0.25))
        al = _results_bits(lb.align(pl, True, 2.5, raw=True)[:len(pl)])
        if with_map:
            maps.append(lb.mapCloudGenerate(all_ids[::-1], I, 0.05))
        best, ld = lb.loopDetect(pl, [0, 3, len(pl)], 2.5, 0.5, raw=True)
        if with_map:
            maps.append(lb.mapCloudGenerate(all_ids, I, 0.0))
        fit = lb.calcFitnessScore([(ids[t], ids[s], G) for s, t, G in pairs], 2.0)
        if with_map:
            lb.removeCloud(extra[1])
            with pytest.raises(pkg.B2RError) as e:
                lb.mapCloudGenerate([ids[0], extra[1]], [np.eye(4)] * 2, 0.25)
            assert e.value.code == _capi.B2R_EINVAL and "unknown cloud id" in str(e.value)
            with pytest.raises(pkg.B2RError):
                lb.mapCloudGenerate([ids[0], 999], [np.eye(4)] * 2, 0.25)
        lb.close()
        return al, best, _results_bits(ld[:len(pl)]), fit.tobytes(), maps

    a, b = run(False), run(True)
    assert a[:4] == b[:4]
    assert all(m.shape[0] > 0 for m in b[4])


@pytest.fixture(scope="module")
def map_scale(synth):
    """250 keyframes of 16 384 points around the circuit (about 4.1 M points), empty keyframes first, in between and last"""
    kfs = [(EMPTY, synth.pose_matrix(0))]
    for f in range(250):
        c = synth.scan("vlp16_16k", frame=f, stride=8)
        if f % 50 == 7:
            c = decorate(c, seed=f)
        kfs.append((c, synth.pose_matrix(f) @ perturb(f, 0.05, 0.5)))
        if f % 61 == 3:
            kfs.append((EMPTY, synth.pose_matrix(f)))
    kfs.append((EMPTY, synth.pose_matrix(3)))
    return kfs


def test_map_scale_equals_host_entry_point(map_scale):
    lb = pkg.RegistrationBatch(params=GICP)
    ids = [lb.addCloud(c) for c, _ in map_scale]
    poses = [P for _, P in map_scale]
    assert sum(c.shape[0] for c, _ in map_scale) > 4000000
    want = lb.engine.mapCloudGenerate(map_scale, 0.05)
    same_rows(lb.mapCloudGenerate(ids, poses, 0.05), want)
    lb.close()


def test_map_too_deep_for_the_octree_keys_is_an_error(synth):
    """at 1 mm resolution two keyframes 3 km apart need more than 21 octree levels: an error, and the batch stays usable"""
    c = synth.scan("vlp16_16k", frame=0, stride=8)[:200].copy()
    far = np.eye(4)
    far[0, 3] = 3000.0
    lb = pkg.RegistrationBatch(params=GICP)
    a = lb.addCloud(c)
    with pytest.raises(pkg.B2RError) as e:
        lb.mapCloudGenerate([a, a], [np.eye(4), far], 0.001)
    assert e.value.code == _capi.B2R_EUNSUPPORTED and "21 octree levels" in str(e.value)
    same_rows(lb.mapCloudGenerate([a], [np.eye(4)], 0.001), lb.engine.mapCloudGenerate([(c, np.eye(4))], 0.001))
    assert lb.align([(a, a, np.eye(4))])[0]["converged"]
    lb.close()
