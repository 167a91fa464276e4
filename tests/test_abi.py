"""CPU-only: the C-ABI library loads and exports every symbol include/b200reg.h declares; without a GPU it refuses to
create a handle (no CPU fallback); the product never links or loads the oracle."""
import os
import re
import shutil
import subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_are_exported():
    from hdl_graph_slam_b200 import build, _capi
    build.build_engine()
    lib = _capi.load()
    hdr = open(os.path.join(ROOT, "include", "b200reg.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(b2r_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in b200reg.h but not exported"
    assert names == {s[0] for s in _capi.SYMBOLS}
    assert b"sm_90a" in lib.b2r_version()


def test_struct_layouts_match_header(tmp_path):
    """sizeof() of every ABI struct as the C compiler sees the header == the ctypes mirror"""
    import ctypes as C
    from hdl_graph_slam_b200 import _capi
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "b200reg.h"\nint main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(b2r_config), sizeof(b2r_result),'
                   ' sizeof(b2r_odometry_params), sizeof(b2r_odometry_status), sizeof(b2r_pair));return 0;}\n')
    exe = tmp_path / "sz"
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    subprocess.check_call([cc, "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    sizes = [int(x) for x in subprocess.run([str(exe)], capture_output=True, text=True).stdout.split()]
    assert sizes == [C.sizeof(_capi.Config), C.sizeof(_capi.Result), C.sizeof(_capi.OdometryParams), C.sizeof(_capi.OdometryStatus), C.sizeof(_capi.Pair)]
    assert C.sizeof(_capi.Result) == 80          # the record all-gathered across GPUs


def test_no_gpu_means_loud_failure_not_fallback():
    import ctypes as C
    from hdl_graph_slam_b200 import _capi
    lib = _capi.load()
    cfg = _capi.Config()
    assert lib.b2r_config_default(C.byref(cfg), 0) == 0
    assert lib.b2r_config_default(C.byref(cfg), 7) == _capi.B2R_EINVAL
    lib.b2r_config_default(C.byref(cfg), 0)
    h = C.c_void_p()
    rc = lib.b2r_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        lib.b2r_destroy(h)
        pytest.skip("a CUDA device is present")
    assert rc == _capi.B2R_ENODEVICE and not h.value and b"CUDA" in lib.b2r_last_error()
    # unsupported registration methods are refused by the factory before any device work
    keys = (C.c_char_p * 1)(b"registration_method")
    vals = (C.c_char_p * 1)(b"GICP_OMP")
    assert lib.b2r_select_registration_method(keys, vals, 1, 0, C.byref(h)) == _capi.B2R_EUNSUPPORTED


def test_product_does_not_touch_the_oracle():
    so = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib", "libb200reg.so")
    out = subprocess.run(["ldd", so], capture_output=True, text=True).stdout
    assert "oracle" not in out
    for dirpath, _, files in os.walk(os.path.join(ROOT, "hdl_graph_slam_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".c", ".h")):
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                assert "liboracle" not in txt and "from oracle" not in txt and "import oracle" not in txt, f


def _f64_ops_of_kernel(ptx_text, mangled_prefix):
    """(op, modifiers) of every float64 multiply / add / subtract / fma in the PTX body of one kernel"""
    i = ptx_text.index(".entry " + mangled_prefix)
    body = ptx_text[i:ptx_text.index("\n}\n", i)]
    return re.findall(r"\b(fma|mad|mul|add|sub)((?:\.\w+)*)\.f64\b", body)


@pytest.fixture(scope="module")
def engine_ptx(tmp_path_factory):
    """the PTX of the engine, compiled with the library's own flags"""
    from hdl_graph_slam_b200 import build
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    ptx = tmp_path_factory.mktemp("ptx") / "api.ptx"
    flags = [f for f in build.NVCC_FLAGS if f not in ("-shared", "-Xcompiler", "-fPIC", "-lineinfo")]
    flags = [f.replace("code=sm_90a", "code=compute_90a") for f in flags]
    subprocess.check_call([nvcc] + flags + ["-ptx", "-o", str(ptx), os.path.join(ROOT, "hdl_graph_slam_b200", "csrc", "api.cu")])
    return ptx.read_text()


def test_voxel_finalize_is_not_contracted(engine_ptx):
    """k_vox_finalize decides a voxel's validity on the sign of its smallest eigenvalue, which for a planar or linear voxel is
    rounding noise: its float64 arithmetic must be the oracle's unfused sequence.  In the PTX of the engine every float64
    multiply / add / subtract of the kernel carries an explicit .rn (which ptxas never fuses) and there is no fma.  The SASS of
    the built library can still hold DFMA: correctly rounded float64 division and square root are DFMA sequences, and those
    round exactly like the oracle's / and sqrt."""
    from hdl_graph_slam_b200 import build
    ops = _f64_ops_of_kernel(engine_ptx, "_ZN3b2r14k_vox_finalize")
    assert len(ops) > 100  # the eigen-solve is in the kernel
    assert not [o for o in ops if o[0] in ("fma", "mad")], "contracted float64 in k_vox_finalize"
    assert not [o for o in ops if ".rn" not in o[1]], "float64 arithmetic without .rn (ptxas may fuse it) in k_vox_finalize"
    # the built library holds the kernel as sm_90a SASS
    build.build_engine()
    so = os.path.join(ROOT, "hdl_graph_slam_b200", "_lib", "libb200reg.so")
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cuobjdump, "-sass", so], capture_output=True, text=True, check=True).stdout
    fins = [f for f in sass.split("Function : ") if f.startswith("_ZN3b2r14k_vox_finalize")]
    assert len(fins) == 1 and "DMUL" in fins[0]


@pytest.mark.parametrize("kernel,min_ops", [("_ZN3b2r13k_map_centers", 9), ("_ZN3b2r10k_map_keys", 3)])
def test_map_cloud_voxel_arithmetic_is_not_contracted(engine_ptx, kernel, min_ops):
    """The map cloud's voxel keys (point - min) / resolution and centres ((key + 0.5) * resolution) + min are float64 expressions
    the oracle rounds after every operation; a multiply-add contracted into one fma rounds once and can move a centre.  The
    kernels' PTX holds no fma and only explicitly rounded (.rn) float64 multiply / add / subtract."""
    ops = _f64_ops_of_kernel(engine_ptx, kernel)
    assert len(ops) >= min_ops  # three axes: add, mul, add each (centres) / sub each (keys)
    assert not [o for o in ops if o[0] in ("fma", "mad")], f"contracted float64 in {kernel}"
    assert not [o for o in ops if ".rn" not in o[1]], f"float64 arithmetic without .rn (ptxas may fuse it) in {kernel}"


def test_pcd_header_parser_runs_without_gpu(tmp_path):
    """b2r_pcd_read_header is host-only: layout of the binary PCD KeyFrame::save writes (packed x y z intensity, 16-byte step)"""
    import ctypes as C
    from hdl_graph_slam_b200 import _capi
    lib = _capi.load()
    p = tmp_path / "c.pcd"
    p.write_bytes(b"# .PCD v0.7\nVERSION 0.7\nFIELDS x y z intensity\nSIZE 4 4 4 4\nTYPE F F F F\nCOUNT 1 1 1 1\nWIDTH 3\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS 3\nDATA binary\n" + bytes(48))
    L, n, off = _capi.PointLayout(), C.c_size_t(), C.c_size_t()
    assert lib.b2r_pcd_read_header(str(p).encode(), C.byref(L), C.byref(n), C.byref(off)) == 0
    assert (L.point_step, L.off_x, L.off_y, L.off_z, L.off_intensity, L.intensity_datatype, n.value) == (16, 0, 4, 8, 12, 7, 3)
    assert off.value == p.stat().st_size - 48
    assert lib.b2r_pcd_read_header(str(tmp_path / "nope.pcd").encode(), C.byref(L), C.byref(n), C.byref(off)) == _capi.B2R_EINVAL
