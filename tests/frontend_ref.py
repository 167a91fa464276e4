"""Reference for the front-end drop-in's message path (adapter/b200_frontend.hpp): what pcl::fromROSMsg produces for pcl::PointXYZI
from an organized sensor_msgs/PointCloud2 whose rows may be padded (row_step > width * point_step).  fromPCLPointCloud2 copies the
message row by row, each row's width records starting at r * row_step, so this applies ingest_ref.decode_pointcloud2 to every row
and stacks the rows; the padding after each row's records is never read.

Also the message builders of the front-end tests: velodyne-style, Ouster-style organized, big-endian, padded and
intensity-less records, each as (fields, point_step, blob) in the shape of sensor_msgs/PointCloud2."""
import numpy as np
from ingest_ref import FLOAT32, NO_FIELD, UINT8, UINT16, decode_pointcloud2

FIELD_SIZE = {1: 1, 2: 1, 3: 2, 4: 2, 5: 4, 6: 4, 7: 4, 8: 8}


def layout_of(fields, point_step, is_bigendian=False):
    """the b2r_point_layout b200_frontend::pointcloud2_layout derives: the first field of each name that is FLOAT32 with count 1 or 0;
    None when x, y or z is missing (the adapter throws std::invalid_argument)"""
    off = {}
    for name in ("x", "y", "z", "intensity"):
        for f in fields:
            if f[0] == name and f[2] == FLOAT32 and f[3] in (0, 1):
                off[name] = f[1]
                break
    if not all(k in off for k in "xyz"):
        return None
    return dict(point_step=point_step, off_x=off["x"], off_y=off["y"], off_z=off["z"], off_intensity=off.get("intensity", NO_FIELD),
                intensity_datatype=FLOAT32, is_bigendian=bool(is_bigendian))


def decode_rows(blob, width, height, row_step, lay):
    """fromROSMsg into PointXYZI for an organized message: width * height records, row-major -> (width * height, 8) uint32"""
    data = np.frombuffer(bytes(blob), np.uint8)
    rows = [decode_pointcloud2(data[r * row_step:r * row_step + width * lay["point_step"]].tobytes(), width, lay) for r in range(height)]
    return np.concatenate(rows) if rows else np.zeros((0, 8), np.uint32)


def message(cloud, kind="velodyne", width=None, height=1, pad=0, big=False, intensity="float32", seed=0):
    """a PointCloud2 of the (n, >=4) float32 `cloud` (x y z intensity): returns dict(fields, point_step, width, height, row_step, data,
    is_bigendian).  kind "velodyne": x y z intensity ring(uint16) time(float32) at point_step 22; "ouster": x y z _ intensity t(uint32)
    reflectivity(uint16) ring(uint8) ambient(uint16) range(uint32) at point_step 48.  `pad` bytes of noise follow every row."""
    cloud = np.asarray(cloud, np.float32)
    n = cloud.shape[0]
    width = n if width is None else width
    assert width * height == n
    rng = np.random.default_rng(seed)
    e = ">" if big else "<"
    if kind == "velodyne":
        point_step = 22
        fields = [("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1), ("intensity", 12, FLOAT32, 1), ("ring", 16, UINT16, 1),
                  ("time", 18, FLOAT32, 1)]
        ioff = 12
    else:
        point_step = 48
        fields = [("x", 0, FLOAT32, 1), ("y", 4, FLOAT32, 1), ("z", 8, FLOAT32, 1), ("intensity", 16, FLOAT32, 1), ("t", 20, 6, 1),
                  ("reflectivity", 24, UINT16, 1), ("ring", 26, UINT8, 1), ("ambient", 28, UINT16, 1), ("range", 32, 6, 1)]
        ioff = 16
    rec = rng.integers(0, 256, size=(n, point_step), dtype=np.uint8)  # every byte the decoder must not read is noise
    for j, off in enumerate((0, 4, 8)):
        rec[:, off:off + 4] = cloud[:, j].astype(e + "f4").view(np.uint8).reshape(n, 4)
    if intensity == "float32":
        rec[:, ioff:ioff + 4] = cloud[:, 3].astype(e + "f4").view(np.uint8).reshape(n, 4)
    elif intensity == "uint8":
        fields = [f if f[0] != "intensity" else ("intensity", ioff, UINT8, 1) for f in fields]
    else:
        fields = [f for f in fields if f[0] != "intensity"]
    row_step = width * point_step + pad
    data = rng.integers(0, 256, size=(height, row_step), dtype=np.uint8)
    data[:, :width * point_step] = rec.reshape(height, width * point_step)
    return dict(fields=fields, point_step=point_step, width=width, height=height, row_step=row_step, data=data.reshape(-1).tobytes(),
                is_bigendian=bool(big))
