"""Build and drive tests/odometry_harness.cpp (adapter/b200_odometry.hpp against the test-only stand-ins): job encoding and answer
decoding, shared by tests/test_odometry_adapter_gpu.py and tools/odometry_adapter_time.py."""
import os
import struct
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ODOMETRY, PREFILTER = 1, 2
OK, INVALID_ARGUMENT, RUNTIME_ERROR = 0, 1, 2


def build_harness(exe):
    from hdl_graph_slam_b200 import build
    build.build_engine()
    lib = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++14", "-O1", "-Wall", "-pthread",
                           "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "hdl_graph_slam_b200", "adapter"), "-o", str(exe),
                           os.path.join(ROOT, "tests", "odometry_harness.cpp"), "-L", lib, "-lb200reg", "-Wl,-rpath," + lib])
    return str(exe)


def _s(s):
    b = s.encode()
    return struct.pack("<i", len(b)) + b


def _kv(d):
    return struct.pack("<i", len(d)) + b"".join(_s(k) + _s(str(v)) for k, v in d.items())


def pcl_input(cloud, width=None, height=1, is_dense=True):
    cloud = np.ascontiguousarray(cloud, np.float32)
    assert cloud.ndim == 2 and cloud.shape[1] == 8
    return ("pcl", cloud, cloud.shape[0] if width is None else width, height, is_dense)


def msg_input(m, is_dense=False):
    return ("msg", m, is_dense)


def encode_call(kind, inp, stamp, frame="velodyne", seq=7, msf=None, want_status=True, want_aligned=True):
    """stamp: (sec, nsec); msf: row-major 4x4 msf_delta or None"""
    if inp[0] == "pcl":
        _, cloud, w, h, dense = inp
        b = struct.pack("<iIII", 0, seq, *stamp) + _s(frame) + struct.pack("<IIiq", w, h, int(dense), cloud.shape[0]) + cloud.tobytes()
    else:
        _, m, dense = inp
        b = struct.pack("<iIII", 1, seq, *stamp) + _s(frame)
        b += struct.pack("<IIIIii", m["width"], m["height"], m["point_step"], m["row_step"], int(m["is_bigendian"]), int(dense))
        b += struct.pack("<i", len(m["fields"])) + b"".join(_s(n) + struct.pack("<IiI", o, t, c) for n, o, t, c in m["fields"])
        b += struct.pack("<q", len(m["data"])) + bytes(m["data"])
    if kind == ODOMETRY:
        T = np.eye(4, dtype=np.float32) if msf is None else np.asarray(msf, np.float32)
        b += struct.pack("<i16f", msf is not None, *T.T.reshape(16))
        b += struct.pack("<ii", int(want_status), int(want_aligned))
    return b


class _R:
    def __init__(self, b):
        self.b, self.o = b, 0

    def get(self, fmt):
        v = struct.unpack_from("<" + fmt, self.b, self.o)
        self.o += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    def str(self):
        n = self.get("i")
        s = self.b[self.o:self.o + n].decode()
        self.o += n
        return s

    def mat(self):
        return np.array(self.get("16f"), np.float32).reshape(4, 4).T.copy()

    def cloud(self):
        if not self.get("i"):
            return None
        seq, stamp = self.get("I"), self.get("Q")
        frame = self.str()
        w, h, dense, n = self.get("IIiq")
        pts = np.frombuffer(self.b, np.uint32, count=n * 8, offset=self.o).reshape(n, 8).copy()
        self.o += n * 32
        return dict(header=(seq, stamp, frame), width=w, height=h, is_dense=bool(dense), bits=pts)


def decode(kind, block):
    """one job's answers: a list of dicts (or ("error", status, text))"""
    r = _R(block)
    out = []
    while r.o < len(block):
        n = r.get("q")
        sub = _R(block[r.o:r.o + n])
        r.o += n
        st = sub.get("i")
        if st != OK:
            out.append(("error", st, sub.str()))
            continue
        if kind == ODOMETRY:
            a = dict(odom=sub.mat(), converged=bool(sub.get("i")), trans=sub.mat(), matching_error=sub.get("d"), inlier_fraction=sub.get("f"),
                     keyframe_updated=bool(sub.get("i")), frame_rejected=bool(sub.get("i")), keyframe_pose=sub.mat())
            a["aligned"] = sub.cloud()
        else:
            a = dict(cloud=sub.cloud())
        out.append(a)
    return out


def run_jobs(harness, tmp_path, jobs, mode="serial", times=False):
    """jobs: [(kind, rosparams, [encoded call, ...])] -> per job its decoded answers (and per job the per-call nanoseconds), plus the
    raw blocks"""
    src, dst, tms = tmp_path / "in.bin", tmp_path / "out.bin", tmp_path / "times.bin"
    src.write_bytes(struct.pack("<i", len(jobs)) + b"".join(struct.pack("<i", k) + _kv(p) + struct.pack("<i", len(c)) + b"".join(c)
                                                             for k, p, c in jobs))
    cmd = [harness, str(src), str(dst), mode] + ([str(tms)] if times else [])
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stderr[-4000:]
    b = dst.read_bytes()
    blocks, o = [], 0
    while o < len(b):
        (n,) = struct.unpack_from("<q", b, o)
        blocks.append(b[o + 8:o + 8 + n])
        o += 8 + n
    answers = [decode(k, blk) for (k, _, _), blk in zip(jobs, blocks)]
    if times:
        t = np.fromfile(str(tms), np.int64)
        per, o = [], 0
        for _, _, c in jobs:
            per.append(t[o:o + len(c)])
            o += len(c)
        return answers, blocks, per
    return answers, blocks
