"""torchrun --nproc-per-node N tools/check_multi_gpu.py [groups] [sensor] [registration_method] — the sharded loop-closure batch (b2r_batch_loop_detect: groups dealt to ranks,
in-library ncclAllGather of 80-byte records) must give EVERY rank the same records, bitwise equal to one GPU aligning all pairs alone
(SURVEY.md §8e "determinism across G")."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist
import hdl_graph_slam_b200 as pkg
from hdl_graph_slam_b200 import synth, batch
from hdl_graph_slam_b200._capi import Pair

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
n_groups = int(sys.argv[1]) if len(sys.argv) > 1 else 6
sensor = sys.argv[2] if len(sys.argv) > 2 else "vlp16_16k"
method = sys.argv[3] if len(sys.argv) > 3 else "FAST_GICP"  # registration_method of both batches (e.g. FAST_VGICP, GICP, B200_VGICP_CUDA, B200_GICP_OMP, B200_NDT_KDTREE)
groups, guesses, group_first = batch.loop_workload(n_groups, sensor)
n_pairs = group_first[-1]


def run(lb, g0, g1):
    needed = sorted({f for g in range(g0, g1) for f in [groups[g][0]] + groups[g][1]})
    ids = {f: lb.addCloud(synth.scan(sensor, frame=f, stride=8)) for f in needed}
    pairs = (Pair * n_pairs)()
    for p in range(n_pairs):
        gc = np.ascontiguousarray(guesses[p].T.reshape(-1))
        for k in range(16):
            pairs[p].guess[k] = gc[k]
        pairs[p].source = pairs[p].target = -1
    for g in range(g0, g1):
        tf, sfs = groups[g]
        for c, sf in enumerate(sfs):
            pairs[group_first[g] + c].source, pairs[group_first[g] + c].target = ids[sf], ids[tf]
    return lb.loopDetect(pairs, group_first, 2.5, 0.5, raw=True)


lb = pkg.RegistrationBatch(params={"registration_method": method}, device_id=local)
idt = torch.zeros(128, dtype=torch.uint8, device=dev)
if rank == 0:
    idt = torch.frombuffer(bytearray(pkg.RegistrationBatch.ncclUniqueId()), dtype=torch.uint8).to(dev)
dist.broadcast(idt, 0)
lb.commInit(bytes(idt.cpu().numpy().tobytes()), rank, world)
g0, g1 = pkg.shard_range(n_groups, world, rank)
best, res = run(lb, g0, g1)
mine = bytes(memoryview(res)[: n_pairs * 80]) + bytes(np.asarray(best, np.int32).tobytes())
# every rank must hold the same bytes
t = torch.frombuffer(bytearray(mine), dtype=torch.uint8).to(dev)
allb = [torch.empty_like(t) for _ in range(world)]
dist.all_gather(allb, t)
same = all(torch.equal(allb[0], x) for x in allb)
ok = same
if rank == 0:
    solo = pkg.RegistrationBatch(params={"registration_method": method}, device_id=local)  # no communicator: one GPU, all pairs
    b1, r1 = run(solo, 0, n_groups)
    ref = bytes(memoryview(r1)[: n_pairs * 80]) + bytes(np.asarray(b1, np.int32).tobytes())
    ok = same and (ref == mine)
    conv = sum(int(r1[i].converged) for i in range(n_pairs))
    print(f"multi-gpu check: world={world} pairs={n_pairs} converged={conv} ranks_agree={same} equals_single_gpu={ref == mine} loops={sum(1 for b in b1 if b >= 0)}", flush=True)
    solo.close()
lb.close()
flag = torch.tensor([1 if ok else 0], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
dist.destroy_process_group()
sys.exit(0 if int(flag.item()) == 1 else 1)
