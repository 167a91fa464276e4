"""GPU: the engine's objects free what they own, and only that.  One cycle touches every lazily allocated workspace of handles,
batches and odometry mirrors and then destroys them all; three cycles run in one process.  Every call must succeed and every cycle
must compute bitwise what the first one did: a double free, a use after free or a buffer freed on the wrong device shows up as an
error or as changed outputs.  Free device memory is not asserted, because the card may be shared with other processes."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CYCLES = 3


def _n_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for l in out.splitlines() if l.startswith("GPU "))
    except Exception:  # noqa: BLE001
        return 0


def _pc2_blob(cloud):
    """PointCloud2 data[]: x y z intensity FLOAT32 at 0, 4, 8, 16, point_step 32"""
    dt = np.dtype({"names": ["x", "y", "z", "intensity"], "formats": ["<f4"] * 4, "offsets": [0, 4, 8, 16], "itemsize": 32})
    rec = np.zeros(cloud.shape[0], dt)
    rec["x"], rec["y"], rec["z"], rec["intensity"] = cloud[:, 0], cloud[:, 1], cloud[:, 2], cloud[:, 4]
    return rec.tobytes(), dict(point_step=32, off_x=0, off_y=4, off_z=8, off_intensity=16, intensity_datatype=7)


def _write_pcd(path, cloud):
    n = cloud.shape[0]
    hdr = ("VERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\n"
           f"WIDTH {n}\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS {n}\nDATA binary\n")
    with open(path, "wb") as f:
        f.write(hdr.encode())
        f.write(np.ascontiguousarray(cloud[:, [0, 1, 2, 4]], np.float32).tobytes())


def _handle(pkg, method, clouds, pcd, out, device_id=0):
    """align with prefetch, fitness, nearest, prefilter (SOR), both voxel grids, ingest, map cloud, NDT voxels, loop matching"""
    tgt, src, nxt = clouds[:3]
    eye = np.eye(4, dtype=np.float32)
    reg = pkg.select_registration_method({"registration_method": method}, device_id=device_id)
    reg.setInputTarget(tgt)
    reg.setInputSource(src)
    reg.prefetchSource(nxt)
    reg.align(eye)
    out += [reg.getFinalTransformation(), np.array(reg.getFitnessScore(2.5, full=True))]
    reg.setInputSource(nxt)  # adopts the prefetched cloud
    reg.align(eye)
    out += [reg.getFinalTransformation(), *reg.nearestKSearch(src[:1000])]
    if method == "NDT_OMP":
        out += list(reg.ndtGetVoxels().values())
    out.append(reg.prefilter(tgt, downsample_resolution=0.2)[0])  # default outlier removal: statistical
    out += [reg.voxelGridFilter(tgt, 0.3), reg.approximateVoxelGridFilter(tgt, 0.3)]
    blob, lay = _pc2_blob(tgt)
    reg.setInputTargetDevice(reg.ingestPointCloud2(blob, tgt.shape[0], **lay), tgt.shape[0], 32)
    out += [*reg.nearestKSearch(src[:1000])]
    dptr, n = reg.ingestPcd(pcd)
    reg.setInputTargetDevice(dptr, n, 32)
    out += [*reg.nearestKSearch(src[:1000])]
    out.append(reg.mapCloudGenerate([(tgt, np.eye(4)), (src, np.eye(4))], 0.5))
    best, res = pkg.LoopDetector(reg, 2.5, 0.5).matching([src, nxt], tgt, [eye, eye])
    out += [np.array([best])] + [np.array([r["fitness"]]) for r in res] + [r["T"] for r in res]
    return reg


def _batch(pkg, method, clouds, out, device_id=0):
    """add, remove and re-add (recycled slots), device-added clouds, align with fitness, calc_fitness_score, map cloud"""
    eye = np.eye(4, dtype=np.float32)
    lb = pkg.RegistrationBatch(params={"registration_method": method}, device_id=device_id)
    ids = [lb.addCloud(c) for c in clouds]
    lb.removeCloud(ids[1])
    lb.removeCloud(ids[3])
    ids[3] = lb.addCloud(clouds[3])  # into the removed clouds' slots and buffers
    ids[1] = lb.addCloud(clouds[1])
    for r in lb.align([(ids[k], ids[0], eye) for k in range(1, len(clouds))], True, 2.5):
        out += [r["T"], np.array([r["fitness"], r["converged"], r["iterations"]])]
    out.append(lb.calcFitnessScore([(ids[0], ids[k], eye) for k in range(1, len(clouds))], 2.5))
    out.append(lb.mapCloudGenerate(ids, [np.eye(4)] * len(ids), 0.5))
    # a device-added cloud: the records of a handle's ingest buffer, the caller's until the align that first uses it returns
    helper = pkg.select_registration_method({"registration_method": "FAST_GICP"}, device_id=device_id)
    blob, lay = _pc2_blob(clouds[2])
    did = lb.addCloudRaw(helper.ingestPointCloud2(blob, clouds[2].shape[0], **lay), clouds[2].shape[0], 32, device=True)
    for r in lb.align([(did, ids[0], eye), (ids[0], did, eye)], True, 2.5):
        out += [r["T"], np.array([r["fitness"], r["converged"], r["iterations"]])]
    helper.close()
    out.append(lb.mapCloudGenerate([did, ids[1]], [np.eye(4)] * 2, 0.5))
    return lb


def _odometry(pkg, clouds, out, close_handle_first):
    """VOXELGRID downsample; the last matching call leaves an announced, unadopted prefetch in flight"""
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    odo = pkg.ScanMatchingOdometry(reg, downsample_method=pkg.B2R_DOWNSAMPLE_VOXELGRID, downsample_resolution=0.2)
    for k, c in enumerate(clouds[:-1]):
        odo.prefetch_raw(clouds[k + 1].ctypes.data, clouds[k + 1].shape[0], clouds[k + 1].shape[1] * 4)
        out.append(odo.matching(0.1 * k, c)["odom"])
    odo.prefetch_raw(clouds[0].ctypes.data, clouds[0].shape[0], clouds[0].shape[1] * 4)
    out.append(odo.matching(0.5, clouds[-1])["odom"])  # prefetches clouds[0], which no call adopts
    if close_handle_first:  # b2r_odometry_destroy must not touch its (destroyed) handle
        reg.close()
        odo.close()
    else:
        odo.close()
        reg.close()


def cycle(pkg, clouds, pcd, n_gpus):
    out = []
    for method in ("FAST_GICP", "NDT_OMP"):
        _handle(pkg, method, clouds, pcd, out).close()
        _batch(pkg, method, clouds, out).close()
    _odometry(pkg, clouds, out, close_handle_first=False)
    _odometry(pkg, clouds, out, close_handle_first=True)
    pkg.select_registration_method({"registration_method": "FAST_GICP"}).close()  # never used
    pkg.RegistrationBatch(params={"registration_method": "NDT_OMP"}).close()
    if n_gpus >= 2:  # objects of device 1, destroyed while device 0 is current, then more work on device 0
        on0 = pkg.select_registration_method({"registration_method": "FAST_GICP"}, device_id=0)
        on1 = _handle(pkg, "FAST_GICP", clouds, pcd, out, device_id=1)
        lb1 = _batch(pkg, "NDT_OMP", clouds, out, device_id=1)
        for obj in (on1, lb1):
            on0.setInputTarget(clouds[0])  # makes device 0 current
            obj.close()
        on0.setInputSource(clouds[1])
        on0.align(np.eye(4, dtype=np.float32))
        out.append(on0.getFinalTransformation())
        on0.close()
    return out


def _same(a, b):
    if a is None or b is None:
        return a is b
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def main(tmpdir):
    sys.path.insert(0, ROOT)
    import hdl_graph_slam_b200 as pkg
    from hdl_graph_slam_b200 import synth
    clouds = [synth.scan("vlp16_16k", frame=f) for f in range(4)]
    pcd = os.path.join(tmpdir, "cloud.pcd")
    _write_pcd(pcd, clouds[0])
    n_gpus = _n_gpus()
    first = cycle(pkg, clouds, pcd, n_gpus)
    for c in range(1, CYCLES):
        got = cycle(pkg, clouds, pcd, n_gpus)
        assert len(got) == len(first)
        bad = [i for i, (a, b) in enumerate(zip(first, got)) if not _same(a, b)]
        assert not bad, f"cycle {c}: outputs {bad} differ from cycle 0"
    print(f"lifecycle ok: {CYCLES} cycles, {len(first)} outputs each, {n_gpus} GPU(s)")


def test_create_use_destroy_cycles_are_repeatable(tmp_path):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "lifecycle ok" in r.stdout


if __name__ == "__main__":
    main(sys.argv[1])
