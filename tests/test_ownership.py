"""Source check: every device, pinned and mapped buffer, stream and event of the engine is owned by a type in csrc/engine.cuh and
freed by its destructor.  Allocating or freeing anywhere else would bring back a hand-written release list, whose forgotten entry is a
leak no other test sees."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "hdl_graph_slam_b200", "csrc")
OWNER = "engine.cuh"
RESOURCE_CALL = re.compile(r"\b(cudaFree|cudaFreeHost|cudaEventDestroy|cudaStreamDestroy|cudaMalloc|cudaMallocHost|cudaHostAlloc)\s*\(|"
                           r"\b(cudaEventCreate|cudaStreamCreate)\w*\s*\(")
# a process-lifetime debug buffer of the B2R_KNN_PROFILE build (not built by default)
ALLOWED = {("api.cu", "if (!d_prof) cudaMalloc(&d_prof, (size_t)(1 << 16) * 8 * sizeof(long long));")}


def _sources():
    for name in sorted(os.listdir(CSRC)):
        with open(os.path.join(CSRC, name)) as f:
            yield name, f.read()


def test_resources_are_allocated_and_freed_only_by_the_owner_types():
    stray = [f"{name}:{i}: {line.strip()}" for name, text in _sources() if name != OWNER
             for i, line in enumerate(text.splitlines(), 1)
             if RESOURCE_CALL.search(line) and (name, line.strip()) not in ALLOWED]
    assert not stray, "allocate / free through the owner types of engine.cuh:\n" + "\n".join(stray)


def test_no_release_lists():
    for name, text in _sources():
        assert not re.search(r"\b(free_cloud|ndt_free_map)\b", text), name
        assert not re.search(r"\brelease\s*\(\s*\)\s*(const\s*)?\{", text), f"{name} defines a release() method"
