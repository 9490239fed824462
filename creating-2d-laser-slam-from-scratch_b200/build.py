"""Build libb200slam.so (CUDA, sm_90a for the H100) in-tree with nvcc.  nvcc cross-compiles without a GPU.
Each source is compiled to an object under csrc/build/ (only when stale, in parallel), then linked."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libb200slam.so")
SOURCES = ["library.cu", "karto_matcher.cu", "karto_occgrid.cu", "hector_map.cu", "hector_slam.cu", "gmapping_map.cu", "plicp.cu", "plicp_odometry.cu", "plicp_scan_match.cu","karto_mapper.cu", "pose_graph.cu", "ros_io.cu", "lidar_undistortion.cu", "pcl_icp.cu", "feature_detection.cu", "lesson4_node_maps.cu", "karto_node.cu", "hector_node.cu"]
HEADERS = ["common.cuh", "scan_kernels.cuh", "glibc_math.cuh", "hector_grid.cuh", "karto_sweep_plan.cuh", "hector_node_plan.cuh", "introsort.cuh", "hector_scan.cuh", "plicp_pair.cuh", "gmapping_grid.cuh", "ros_math.cuh", "karto_internal.cuh", os.path.join("..", "..", "include", "b200slam.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-fmad=false", "-std=c++17",
              "-Xcompiler", "-fPIC"]


def nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def needs_build() -> bool:
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return _stale(LIB, deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    jobs = []
    for s in SOURCES:
        src, obj = os.path.join(CSRC, s), os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs):
            jobs.append([nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj])
    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        for rc in ex.map(lambda cmd: subprocess.run(cmd).returncode, jobs):
            if rc != 0:
                raise RuntimeError("nvcc failed")
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    subprocess.check_call([nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static",
                           "-Xcompiler", "-fPIC"] + objs + ["-o", LIB])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
