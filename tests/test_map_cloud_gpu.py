"""GPU: MapCloudGenerator::generate ("next" row f-3; src/hdl_graph_slam/map_cloud_generator.cpp:13-51) on the device against a numpy
restatement that follows PCL's sequential octree growth: the concatenated transformed cloud bit-exact, the occupied voxel centres
equal bit for bit as a SET — PCL's traversal order is not reproduced (documented in b200reg.h)."""
import numpy as np
import pytest
import hdl_graph_slam_b200 as pkg

pytestmark = pytest.mark.gpu


def keyframes(synth, frames, sensor="vlp16_16k"):
    return [(synth.scan(sensor, frame=f, stride=8), synth.pose_matrix(f)) for f in frames]


def test_unfiltered_map_is_the_transformed_concatenation(synth, oracle):
    kfs = keyframes(synth, (0, 3, 7, 12))
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    got = reg.mapCloudGenerate(kfs, 0.0)
    want = oracle.map_cloud_generate(kfs, 0.0)
    assert got.shape[0] == want.shape[0] == sum(c.shape[0] for c, _ in kfs)
    assert np.array_equal(got[:, :3], want[:, :3]) and np.all(got[:, 3] == 1.0) and np.array_equal(got[:, 4], want[:, 4])
    assert reg.mapCloudGenerate([], 0.1) is None  # "warning: keyframes empty!!"
    reg.close()


@pytest.mark.parametrize("res", [0.05, 0.25, 1.0])
def test_voxel_centres_equal_octree_occupied_centres(synth, oracle, res):
    kfs = keyframes(synth, (0, 5, 10, 60, 130))  # spread over half the circuit: the octree box grows many times
    kfs[1][0][17, 0] = np.nan                      # non-finite points are not inserted
    reg = pkg.select_registration_method({"registration_method": "FAST_GICP"})
    got = reg.mapCloudGenerate(kfs, res)
    want = oracle.map_cloud_generate(kfs, res)
    assert got.shape[0] == want.shape[0] and 0 < got.shape[0] < sum(c.shape[0] for c, _ in kfs)
    g = got[:, :3]
    g = g[np.lexsort((g[:, 0], g[:, 1], g[:, 2]))]
    assert np.array_equal(g, want)  # (key + 0.5) * res + min rounded after the multiply and after the add, as the oracle does
    assert np.all(got[:, 3] == 1.0) and np.all(got[:, 4] == 0.0)
    reg.close()
