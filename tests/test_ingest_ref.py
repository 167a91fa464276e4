"""CPU: known answers for the PointCloud2 reference decoder of tests/ingest_ref.py, on records packed by hand with struct — every
intensity datatype in both byte orders, an odd point_step, and special float bit patterns carried bit for bit."""
import struct
import numpy as np
import pytest
from ingest_ref import NO_FIELD, ONE_BITS, FLOAT32, DATATYPE_SIZE, layout, decode_pointcloud2

_FMT = {1: "b", 2: "B", 3: "h", 4: "H", 5: "i", 6: "I", 7: "f", 8: "d"}
_VAL = {1: -7, 2: 200, 3: -1234, 4: 54321, 5: -123456, 6: 3000000000, 7: 17.25, 8: -2.5}


def _bits(f):
    return struct.unpack("<I", struct.pack("<f", f))[0]


@pytest.mark.parametrize("big", [False, True], ids=["le", "be"])
@pytest.mark.parametrize("dt", list(range(1, 9)))
def test_decoder_maps_only_float32_intensity(dt, big):
    """record of 23 bytes: pad(1) x(@1) y(@5) z(@9) intensity(@13) pad: intensity comes through only as FLOAT32, else 0"""
    e = ">" if big else "<"
    recs = b""
    xyz = [(1.5, -2.0, 3.25), (-0.0, 1e-40, float("inf"))]
    for x, y, z in xyz:
        r = b"\xaa" + struct.pack(e + "fff", x, y, z) + struct.pack(e + _FMT[dt], _VAL[dt])
        recs += r + b"\x55" * (23 - len(r))
    got = decode_pointcloud2(recs, 2, layout(23, 1, 5, 9, 13, dt, big))
    for i, (x, y, z) in enumerate(xyz):
        assert list(got[i, :3]) == [_bits(x), _bits(y), _bits(z)]
        assert got[i, 3] == ONE_BITS and list(got[i, 5:]) == [0, 0, 0]
        assert got[i, 4] == (_bits(_VAL[dt]) if dt == FLOAT32 else 0)


def test_decoder_without_intensity_and_with_special_bits():
    step = 13
    words = [0x7FC00001, 0xFFA00000, 0x80000000, 0x00000001, 0x7F800000, 0xFF800000]  # quiet / signalling NaN payloads, -0, denormal, +-inf
    rec = bytearray()
    for i in range(len(words) - 2):
        rec += struct.pack("<III", words[i], words[i + 1], words[i + 2]) + b"\x01"
    n = len(rec) // step
    got = decode_pointcloud2(bytes(rec), n, layout(step, 0, 4, 8))
    assert np.array_equal(got[:, :3], np.array([words[i:i + 3] for i in range(n)], np.uint32))
    assert np.all(got[:, 4] == 0) and np.all(got[:, 3] == ONE_BITS)
    # the same bytes read as big-endian swap every word
    got_be = decode_pointcloud2(bytes(rec), n, layout(step, 0, 4, 8, is_bigendian=True))
    assert np.array_equal(got_be[:, :3], got[:, :3].byteswap())


def test_decoder_reads_only_n_records_and_overlapping_fields():
    """fields may overlap (intensity inside x), and trailing bytes beyond n records are ignored"""
    rec = struct.pack("<fff", 1.0, 2.0, 3.0)
    got = decode_pointcloud2(rec * 3 + b"\xff" * 7, 3, layout(12, 0, 4, 8, 0, FLOAT32))
    assert np.all(got[:, 4] == got[:, 0]) and got.shape == (3, 8)
    assert decode_pointcloud2(b"", 0, layout(12)).shape == (0, 8)
    assert sorted(DATATYPE_SIZE) == list(range(1, 9)) and NO_FIELD == 0xFFFFFFFF
