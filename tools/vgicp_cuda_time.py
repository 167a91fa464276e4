"""The factory's `FAST_VGICP_CUDA` branch as B200_VGICP_CUDA (B2R_METHOD_VGICP_CUDA) timed beside FAST_VGICP on one GPU.

    python tools/vgicp_cuda_time.py [--frames 40] [--groups 256] [--reps 3] [--out profiles/h100/vgicp_cuda_time_1.json]

The scans, workloads and statistics are tools/vgicp_time.py's (odometry over VLP-16 frames of 65 536 points from host clouds and
HBM-resident, the loop batch of --groups x 8 candidates with fitness, reps alternated between the methods, one profiled pass per method);
only the two methods differ: B200_VGICP_CUDA and FAST_VGICP, both at reg_resolution 1.0.  Prints one JSON record; the card's name, power
limit and clocks are read in the same call.  No speed-up is assumed: the record holds both methods' numbers as measured."""
import contextlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import vgicp_time  # noqa: E402

METHODS = {"B200_VGICP_CUDA": {"registration_method": "B200_VGICP_CUDA", "reg_resolution": "1.0"},
           "FAST_VGICP": {"registration_method": "FAST_VGICP", "reg_resolution": "1.0"}}


def main():
    out = None
    argv = list(sys.argv[1:])
    if "--out" in argv:
        i = argv.index("--out")
        out = argv[i + 1]
        del argv[i:i + 2]
    vgicp_time.METHODS.clear()
    vgicp_time.METHODS.update(METHODS)
    buf = io.StringIO()
    sys.argv = [sys.argv[0]] + argv
    with contextlib.redirect_stdout(buf):
        vgicp_time.main()
    rec = json.loads(buf.getvalue().strip().splitlines()[-1])
    rec["tool"] = "vgicp_cuda_time"
    print(json.dumps(rec))
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
