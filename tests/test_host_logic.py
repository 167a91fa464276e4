"""CPU-only: the engine's exact BVH search logic (bvh.cuh compiled as HOST code by tests/host_harness.cu) returns the
oracle's (d2, index) results bit-for-bit, including lattice ties, range-limited search and queries far outside the cloud; and the
warp-group traversal the kernels actually run (bvh_group_search: group masks, per-lane refinement, centred window, tile /
two-phase / cooperative leaf visits, C lanes per query) does the same when executed on an emulated 32-lane warp
(tests/warp_emu.hpp + tests/warp_harness.cpp)."""
import os
import subprocess
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def harness(oracle):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    exe = os.path.join(ROOT, "build", "host_harness")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-w", "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "tests", "host_harness.cu"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Xlinker", "-rpath=" + os.path.join(ROOT, "oracle")])
    return exe


@pytest.mark.parametrize("mode,n", [(0, 20000), (1, 20000), (2, 20000), (0, 1500)])
def test_bvh_search_equals_kdtree(harness, mode, n):
    out = subprocess.run([harness, str(n), "4000", str(mode)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "1nn_mismatch=0" in out.stdout and "knn_mismatch=0" in out.stdout and "limited_mismatch=0" in out.stdout


def test_min_eigenvector_solver_matches_jacobi(tmp_path):
    exe = tmp_path / "eig_harness"
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-w", "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
                           "-o", str(exe), os.path.join(ROOT, "tests", "eig_harness.cu")])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


def test_voxel_finalize_equals_oracle_bitwise(oracle, tmp_path):
    """The NDT voxel finalisation (ndt_voxel_gaussian: covariance, Jacobi eigen-solve, 1 % clamp, inverse — what k_vox_finalize runs)
    and its eigen-solver sym_eigen3 alone, compiled as host code, against the oracle's orc_ndt_voxel_gaussian / orc::sym_eigen<3> on
    1e5 voxels of 5-15 points on exact planes and lines, all-identical points, generic and nearly planar voxels, at the origin and
    shifted by (2e4, -3e4, 50): npts, mean, icov, eigenvalues and eigenvectors bit-identical."""
    exe = tmp_path / "vox_eig_harness"
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-w", "-Wno-deprecated-gpu-targets", "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
                           "-Xcompiler", "-ffp-contract=off", "-o", str(exe), os.path.join(ROOT, "tests", "vox_eig_harness.cu"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Xlinker", "-rpath=" + os.path.join(ROOT, "oracle")])
    out = subprocess.run([str(exe), "100000"], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "eig_mismatch=0" in out.stdout and "gauss_mismatch=0" in out.stdout
    # the cases reach every branch: invalidated voxels, one and two clamped eigenvalues
    stats = dict(kv.split("=") for kv in out.stdout.split() if "=" in kv)
    assert int(stats["invalid"]) > 1000 and int(stats["clamped_one"]) > 1000 and int(stats["clamped_two"]) > 1000


@pytest.fixture(scope="module")
def warp_harness(oracle):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    exe = os.path.join(ROOT, "build", "warp_harness")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.check_call(["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++17", "-O1", "-w", "-ffp-contract=off", "-I" + cuda_inc,
                           "-o", exe, os.path.join(ROOT, "tests", "warp_harness.cpp"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Wl,-rpath=" + os.path.join(ROOT, "oracle")])
    return exe


@pytest.mark.parametrize("mode,copies", [(0, 1), (0, 2), (0, 4), (0, 8), (1, 1), (1, 4), (2, 4)])
def test_warp_group_traversal_on_emulated_warp(warp_harness, mode, copies):
    """1-NN (unseeded / seeded / hinted / range-limited / straddling groups / inactive lanes) and 20-NN of a cloud against itself:
    every result equals the oracle's exact (d2, index) answer; copies of one query agree; lanes never diverge around a collective."""
    out = subprocess.run([warp_harness, "6000", "24", str(mode), str(copies)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "1nn_mismatch=0" in out.stdout and "knn_mismatch=0" in out.stdout


@pytest.mark.parametrize("n", [1, 5, 33, 1024, 1025, 2049])
def test_warp_group_traversal_edge_sizes(warp_harness, n):
    """clouds of 1 point, less than a leaf, one leaf + 1, exactly one super-node, one super-node + 1, two + 1 — on the lattice (ties)"""
    out = subprocess.run([warp_harness, str(n), "8", "1", "4"], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "1nn_mismatch=0" in out.stdout and "knn_mismatch=0" in out.stdout


@pytest.mark.parametrize("copies", [1, 4])
def test_warp_group_traversal_on_lidar_scans(warp_harness, synth, tmp_path, copies):
    """same check on two real synthetic VLP-16 scans (rings, sparse far field) related by the odometry guess of the trajectory"""
    import numpy as np
    tgt = synth.scan("vlp16_16k", frame=5, stride=4)
    src = synth.scan("vlp16_16k", frame=7, stride=4)
    rel = (np.linalg.inv(synth.pose_matrix(5)) @ synth.pose_matrix(6)).astype(np.float32)  # guess: the previous frame's pose
    tgt.tofile(tmp_path / "t.f32")
    src.tofile(tmp_path / "s.f32")
    out = subprocess.run([warp_harness, str(tgt.shape[0]), "24", "3", str(copies), str(tmp_path / "t.f32"), str(tmp_path / "s.f32")]
                         + [repr(float(x)) for x in rel[:3, :].reshape(-1)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "1nn_mismatch=0" in out.stdout and "knn_mismatch=0" in out.stdout


def test_result_message_protocol(tmp_path):
    """the fence-free result publication (engine.cuh): a message is accepted iff flag, checksum and all words are of the same launch,
    for every order in which the stores can land"""
    exe = tmp_path / "msg_harness"
    subprocess.check_call(["nvcc", "-O1", "-std=c++17", "-w", "-Wno-deprecated-gpu-targets", "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
                           "-o", str(exe), os.path.join(ROOT, "tests", "msg_harness.cu")])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "accepted_partial=0" in out.stdout and "rejected_complete=0" in out.stdout


@pytest.fixture(scope="module")
def lm_harness(oracle):
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    exe = os.path.join(ROOT, "build", "lm_harness")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-w", "-gencode", "arch=compute_90a,code=sm_90a", "-ccbin", "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++",
                           "-Xcompiler", "-ffp-contract=off", "-o", exe, os.path.join(ROOT, "tests", "lm_harness.cu"),
                           "-L" + os.path.join(ROOT, "oracle"), "-loracle", "-Xlinker", "-rpath=" + os.path.join(ROOT, "oracle")])
    return exe


@pytest.mark.parametrize("case", ["odometry", "loop_perturbed", "iteration_cap", "far_guess", "tight_epsilon"])
def test_device_lm_state_machine_equals_oracle_step_lm(lm_harness, synth, tmp_path, case):
    """The LM step the GPU runs in k_pair_accumulate's last block (pair_engine.cuh: lm_advance / lm_propose / lm_begin_outer), driven on
    the CPU with the oracle's linearize / compute_error as the two kernels of a round: same iterations, trials, convergence flag,
    final pose and last correspondences as the oracle's own LsqRegistration loop — including rejected trials (rho < 0), the
    iteration cap and the 'converged by a rejected tiny step' exit."""
    import numpy as np
    from common import perturb
    tgt = synth.scan("vlp16_16k", frame=5, stride=4)
    src = synth.scan("vlp16_16k", frame=7 if case != "loop_perturbed" else 9, stride=4)
    max_it, eps, dist = 64, 0.01, 2.5
    guess = np.eye(4)
    if case == "loop_perturbed":
        guess = np.linalg.inv(synth.pose_matrix(5)) @ synth.pose_matrix(9) @ perturb(3, 0.5, 3.0)
    elif case == "iteration_cap":
        max_it = 2
    elif case == "far_guess":
        guess = perturb(11, 2.0, 8.0)  # many correspondences beyond 2.5 m: rejected trials and lambda growth
    elif case == "tight_epsilon":
        eps = 1e-5
    tgt.tofile(tmp_path / "t.f32")
    src.tofile(tmp_path / "s.f32")
    g = np.asarray(guess, np.float32)
    out = subprocess.run([lm_harness, str(tmp_path / "s.f32"), str(tmp_path / "t.f32"), "4", str(max_it), repr(eps), repr(dist)]
                         + [repr(float(x)) for x in g.reshape(-1)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "mismatches=0" in out.stdout
