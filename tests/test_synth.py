"""CPU: the synthetic LiDAR generator refuses scan shapes its fixed beam table cannot hold instead of writing past it."""
import ctypes as C
import numpy as np
import pytest


def test_ring_count_beyond_the_beam_table_is_rejected(synth):
    lib = synth._load()
    n_az, stride = 8, 4
    # a buffer large enough for the requested shape: a generator that ignored its limit would fill it (and overrun elev[64])
    buf = np.full((128 * n_az, stride), -7.0, np.float32)
    for rings in (65, 128, 1, 0, -3):
        assert lib.b2s_scan(rings, n_az, 0.0, 0.0, 0.0, 0.0, 0.0, 1, 0.02, buf.ctypes.data_as(C.c_void_p), stride) == 0
        assert np.all(buf == -7.0), f"{rings} rings: the generator wrote points"
    assert lib.b2s_scan(16, 0, 0.0, 0.0, 0.0, 0.0, 0.0, 1, 0.02, buf.ctypes.data_as(C.c_void_p), stride) == 0
    for shape in ((128, 2048), (65, 16), (1, 16)):
        with pytest.raises(ValueError):
            synth.scan(shape, frame=0)


def test_sixty_four_rings_fill_the_whole_scan(synth):
    c = synth.scan((64, 4096), frame=2, stride=4)
    assert c.shape == (262144, 4) and np.all(np.isfinite(c)) and np.all(c[:, 3] == 1.0)
    r = np.linalg.norm(c[:, :3], axis=1)
    assert r.min() >= 0.25 and r.max() < 120.0  # every ray hits the closed world
    assert np.array_equal(c, synth.scan((64, 4096), frame=2, stride=4))  # seeded: the same frame twice is the same scan
