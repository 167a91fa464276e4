"""CPU: the sequential reference of pcl::ApproximateVoxelGrid (tests/approx_voxelgrid_ref.cpp) against an independent numpy
restatement written from the filter's description (DESIGN.md §2), against the voxel-grid oracle where the two filters must agree, and
its pinned float -> int conversion against this host's own."""
import platform

import numpy as np
import pytest

from approx_voxelgrid_ref import Reference, CASES, case, records, same_bits

INT_MIN = -(2 ** 31)


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    return Reference(tmp_path_factory.mktemp("avg_ref"))


def restated(cloud, leaf):
    """ApproximateVoxelGrid's walk with numpy float32 scalars: 512 history slots, a colliding cell flushes its slot, then the
    remaining slots in slot order.  Shares nothing with the C++ reference."""
    f = np.float32
    inv = f(1.0) / f(leaf)
    c = np.asarray(cloud, np.float32)
    stride = c.shape[1]

    def to_int(v):  # cvttss2si: truncation, INT_MIN for NaN, +-inf and anything outside int32
        return int(v) if (v >= f(-2147483648.0) and v < f(2147483648.0)) else INT_MIN

    slots = [None] * 512
    out, counts = [], []

    def emit(s):
        cnt = f(s[4])
        rec = np.zeros(stride, np.float32)
        rec[0], rec[1], rec[2] = s[3][0] / cnt, s[3][1] / cnt, s[3][2] / cnt
        if stride >= 4:
            rec[3] = 1.0
        if stride >= 5:
            rec[4] = s[3][3] / cnt
        out.append(rec)
        counts.append(s[4])

    with np.errstate(all="ignore"):
        for row in c:
            cell = tuple(to_int(np.floor(row[d] * inv)) for d in range(3))
            h = ((cell[0] * 7171 + cell[1] * 3079 + cell[2] * 4231) & 0xFFFFFFFF) & 511
            s = slots[h]
            if s is not None and s[:3] != cell:
                emit(s)
                s = None
            if s is None:
                s = (cell[0], cell[1], cell[2], [f(0), f(0), f(0), f(0)], 0)
            acc = s[3]
            acc[0] = acc[0] + row[0]
            acc[1] = acc[1] + row[1]
            acc[2] = acc[2] + row[2]
            acc[3] = acc[3] + (row[4] if stride >= 5 else f(0))
            slots[h] = (s[0], s[1], s[2], acc, s[4] + 1)
        for s in slots:
            if s is not None:
                emit(s)
    o = np.array(out, np.float32).reshape(-1, stride)
    return o, np.array(counts, np.int32)


def check_same(ref, cloud, leaf):
    got, cnt = ref.approximate_voxelgrid(cloud, leaf)
    want, wcnt = restated(cloud, leaf)
    assert same_bits(got, want)
    assert np.array_equal(cnt, wcnt)
    assert cnt.sum() == cloud.shape[0]
    return got, cnt


@pytest.mark.parametrize("leaf", [0.1, 0.25, 1.0])
def test_reference_equals_restatement_on_a_scan(ref, synth, leaf):
    cloud = synth.scan("vlp16_16k", frame=3, stride=8)
    got, cnt = check_same(ref, cloud, leaf)
    assert got.shape[0] < cloud.shape[0]


@pytest.mark.parametrize("name", CASES)
def test_reference_equals_restatement_on_edge_cases(ref, name):
    cloud, leaf = case(name)
    got, cnt = check_same(ref, cloud, leaf)
    if name == "same_bucket_alternating":  # every point after the first flushes the other cell's single point
        assert got.shape[0] == cloud.shape[0] and np.all(cnt == 1)
    elif name == "one_cell":
        assert got.shape[0] == 1 and cnt[0] == cloud.shape[0]
    elif name == "every_bucket":  # no collision: the outputs come in slot order, not input order
        assert got.shape[0] == 512 and not np.array_equal(got[:, 0], cloud[:, 0])
    elif name == "nonfinite":
        assert np.isnan(got[:, :3]).any()


def test_distinct_buckets_give_the_voxel_grid(ref, oracle):
    """Cells that all hash to different buckets never collide: every cell is flushed once, in slot order, with its points summed in
    ascending index, so the outputs sorted are exactly the voxel grid's (which also sums a voxel in ascending index)."""
    rng = np.random.default_rng(5)
    cells = np.c_[rng.permutation(512)[:300], np.zeros(300), np.zeros(300)]   # (i, 0, 0): distinct buckets (7171 is odd)
    pts = cells[rng.integers(0, 300, 5000)] + rng.uniform(0.0, 0.999, (5000, 3))
    cloud = records(pts * 0.5, 8)
    got, cnt = ref.approximate_voxelgrid(cloud, 0.5)
    vg, _, vcnt, rc = oracle.voxelgrid(cloud, 0.5)
    assert rc == 0 and got.shape[0] == vg.shape[0] == 300
    mine = np.c_[got[:, :3], got[:, 4]]
    order = np.lexsort((mine[:, 0],))
    vorder = np.lexsort((vg[:, 0],))
    assert np.array_equal(mine[order].view(np.uint32), vg[vorder].view(np.uint32))
    assert np.array_equal(cnt[order], vcnt[vorder])


def test_pinned_conversion_is_the_hosts(ref):
    """static_cast<int> of NaN, +-inf and +-3e9 on this x86 host == the rule the engine emulates (INT_MIN for all of them)"""
    if platform.machine() not in ("x86_64", "AMD64"):
        pytest.skip("the pinned rule is x86's cvttss2si")
    vals = [float("nan"), float("inf"), float("-inf"), 3e9, -3e9, 2147483648.0, -2147483648.0, 2147483520.0, -2147483520.0, -1.5, 2.75]
    for v in vals:
        assert ref.lib.ref_x86_cvtt(v) == ref.lib.ref_static_cast_int(v), v
    with np.errstate(invalid="ignore"):
        assert np.array_equal(np.array(vals, np.float32).astype(np.int32), [ref.lib.ref_x86_cvtt(v) for v in vals])
    assert [ref.lib.ref_x86_cvtt(v) for v in vals[:6]] == [INT_MIN] * 6
