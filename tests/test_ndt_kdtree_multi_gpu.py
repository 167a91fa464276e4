"""GPU (>= 2 devices): an NDT_OMP KDTREE (B2R_METHOD_NDT_KDTREE) loop-closure batch sharded over an NCCL communicator (b2r_batch_loop_detect) gives every rank the same
records, bitwise equal to one GPU aligning all pairs.  Skipped on a 1-GPU box (the single-rank b2r_batch_loop_detect == b2r_batch_align
check runs in tests/test_ndt_kdtree_switches_gpu.py); tools/check_multi_gpu.py is the torchrun body."""
import os
import subprocess
import sys
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _n_gpus():
    try:
        out = subprocess.run(["nvidia-smi", "-L"], capture_output=True, text=True, timeout=30).stdout
        return sum(1 for l in out.splitlines() if l.startswith("GPU "))
    except Exception:  # noqa: BLE001
        return 0


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_ndt_kdtree_batch_is_bitwise_equal_to_single_gpu(world):
    if _n_gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
                        "--master-port", str(29780 + world), os.path.join(ROOT, "tools", "check_multi_gpu.py"), "6", "vlp16_16k", "B200_NDT_KDTREE"],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "equals_single_gpu=True" in r.stdout and "ranks_agree=True" in r.stdout
