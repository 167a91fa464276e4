"""One pass over the FastVGICPCuda (B200_VGICP_CUDA) code the diagnostic switches select, run in a fresh process per configuration (the engine reads each switch
once per process): a FastVGICPCuda odometry chain with the next frame announced (single-pair rounds, PDL, the report wait), and a 24-pair FastVGICPCuda
loop batch with fitness (two lanes under B2R_BATCH_LANES=2, several chunks under B2R_BATCH_CHUNK) through b2r_batch_align and the
single-rank b2r_batch_loop_detect.  Prints, as its last line, one JSON object: a SHA-1 per output, and the raw batch records of both entry
points so that tests/test_vgicp_cuda_switches_gpu.py can compare them.  Used as `python tests/vgicp_cuda_switch_workload.py`."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]

import hdl_graph_slam_b200 as pkg  # noqa: E402
from hdl_graph_slam_b200 import synth, batch  # noqa: E402
from switch_workload import sha, status_rows  # noqa: E402

VGICP = {"registration_method": "B200_VGICP_CUDA", "reg_resolution": "1.0"}


def records(res):
    return np.stack([np.concatenate([np.asarray(r["T"], np.float32).reshape(-1).view(np.uint32).astype(np.uint64),
                                     [np.float64(r["fitness"]).view(np.uint64), r["converged"], r["iterations"]]]).astype(np.uint64) for r in res])


def run():
    out = {}
    # ---- odometry: VLP-16 frames (65 536 points), every next frame announced
    frames = [synth.scan("vlp16", frame=k, stride=8) for k in range(6)]
    reg = pkg.select_registration_method(VGICP)
    odo = pkg.ScanMatchingOdometry(reg, keyframe_delta_trans=0.25, publish_status=True)
    sts = []
    for k, c in enumerate(frames):
        if k + 1 < len(frames):
            nxt = frames[k + 1]
            odo.prefetch_raw(nxt.ctypes.data, nxt.shape[0], nxt.shape[1] * 4)
        sts.append(odo.matching(0.1 * k, c))
    odo.close()
    reg.close()
    out["odometry"] = sha(status_rows(sts), np.array([s["matching_error"] for s in sts]))
    # ---- loop batch: 3 keyframe groups x 8 candidates of 16 384-point scans
    groups, guesses, group_first = batch.loop_workload(3, "vlp16_16k")
    lf = sorted({f for tf, sfs in groups for f in [tf] + list(sfs)})
    lb = pkg.RegistrationBatch(params=VGICP)
    ids = {f: lb.addCloud(synth.scan("vlp16_16k", frame=f, stride=8)) for f in lf}
    pairs = [(ids[sf], ids[tf], guesses[group_first[g] + c]) for g, (tf, sfs) in enumerate(groups) for c, sf in enumerate(sfs)]
    aligned = records(lb.align(pairs, True, 2.5))
    best, det = lb.loopDetect(pairs, group_first, 2.5, 0.5)
    detected = records(det)
    lb.close()
    out["batch_align"] = sha(aligned)
    out["loop_detect"] = sha(detected, np.asarray(best, np.int64))
    print(json.dumps(dict(outputs=out, batch_align=aligned.tolist(), loop_detect=detected.tolist(), best=[int(b) for b in best],
                          group_first=[int(x) for x in group_first])))


if __name__ == "__main__":
    run()
