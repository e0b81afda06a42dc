# SPDX-License-Identifier: Apache-2.0
"""In-tree build of ``libupkie_b200.so`` with nvcc for sm_90a (H100)."""

import os
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libupkie_b200.so")
# compiled in parallel, then linked; the step_*.cu units hold the step kernels of one TILE of one or two families each
# (csrc/step_family.h)
SOURCES = ["upkie_b200.cu", "step_device.cu", "step_host.cu", "step_multicast.cu", "step_device_limits.cu",
           "step_host_limits.cu", "step_multicast_limits.cu", "step_device_spine.cu", "step_host_spine.cu",
           "step_device_body.cu", "step_host_body.cu", "step_device_table.cu", "step_host_table.cu", "base_velocity.cu",
           "reset_randomization.cu", "pushes.cu", "step_device_push.cu", "step_host_push.cu",
           "step_device_body_push.cu", "step_host_body_push.cu"]
DEPS = SOURCES + ["base_velocity.cuh", "base_velocity_core.cuh",
    "sim_core.cuh", "sim_pair.cuh", "kernel_common.cuh", "step_kernel.cuh", "step_family.h", "params.h", "mpc.cuh",
    "mpc_core.cuh",
    "observers.cuh", "observers_core.cuh", "controllers.cuh", "controllers_core.cuh", "../../include/upkie_b200.h",
]

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + [
    "-lineinfo", "-O3", "-std=c++17",
    # approximate division / sqrt / sincos (<= 2 ulp, arguments range-reduced in the code) and FTZ; the parity
    # tolerances already absorb fp32 round-off of that size (bench.py's exact_mode line times the library without it)
    "--use_fast_math",
    "-Xcompiler", "-fPIC",
]
# translation units built without --use_fast_math: the base-velocity epilogue reproduces torch's IEEE cos / sin and
# unfused fp32 products bit for bit (csrc/base_velocity_core.cuh)
IEEE_SOURCES = {"base_velocity.cu"}


def _flags(src: str, flags: list) -> list:
    return [f for f in flags if f != "--use_fast_math"] if src in IEEE_SOURCES else flags


def source_hash() -> str:
    """sha256 (first 16 hex digits) over the CUDA sources and compile flags of the library: the key that ties a
    committed ncu sidecar (``profiles/ncu_sidecar.json``, written by ``tools/ncu_summary.py``) to the build that is
    benchmarked. Stable across rebuilds and machines, unlike a hash of the binary."""
    import hashlib

    h = hashlib.sha256()
    for d in sorted(DEPS):
        with open(os.path.join(CSRC, d), "rb") as f:
            h.update(d.encode() + b"\0" + f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()[:16]


def is_stale() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


# ---- exact-arithmetic build (test / measurement companion of the product library) ------------------------------------
# Same sources WITHOUT --use_fast_math (IEEE division / sqrt / sincos, no flush-to-zero), device-buffer kernels only
# (TILE=0: plain, extras, extras + limits); the step dispatch reports the other families as cudaErrorNotSupported.
# Used by tests/test_gpu_exact_mode.py and bench.py's `exact_mode` line: what the one shortcut of the timed kernel
# (fast-math) costs in accuracy and buys in time.
EXACT_LIB_PATH = os.path.join(_HERE, "libupkie_b200_exact.so")
EXACT_SOURCES = ["upkie_b200.cu", "step_device.cu", "step_device_limits.cu", "exact_stubs.cu", "base_velocity.cu",
                 "reset_randomization.cu", "pushes.cu"]
EXACT_FLAGS = [f for f in NVCC_FLAGS if f != "--use_fast_math"] + ["-DUPKIE_EXACT_BUILD=1"]


def exact_is_stale() -> bool:
    if not os.path.exists(EXACT_LIB_PATH):
        return True
    t = os.path.getmtime(EXACT_LIB_PATH)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS + ["exact_stubs.cu"])


def build_exact(force: bool = False) -> str:
    if not force and not exact_is_stale():
        return EXACT_LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    objdir = os.path.join(_HERE, "build", "exact")
    os.makedirs(objdir, exist_ok=True)
    objs, procs = [], []
    for src in EXACT_SOURCES:
        obj = os.path.join(objdir, os.path.splitext(src)[0] + ".o")
        objs.append(obj)
        procs.append(subprocess.Popen([nvcc] + EXACT_FLAGS + ["-c", "-o", obj, os.path.join(CSRC, src)]))
    failed = [src for src, p in zip(EXACT_SOURCES, procs) if p.wait() != 0]
    if failed:
        raise RuntimeError(f"nvcc (exact build) failed on {failed}")
    subprocess.check_call([nvcc] + GENCODE + ["-shared", "-o", EXACT_LIB_PATH] + objs)
    return EXACT_LIB_PATH


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA library (cross-compiles without a GPU)."""
    if not force and not is_stale():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "nvcc")
    flags = NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else [])
    objdir = os.path.join(_HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs, procs = [], []
    for src in SOURCES:
        obj = os.path.join(objdir, os.path.splitext(src)[0] + ".o")
        objs.append(obj)
        procs.append(subprocess.Popen([nvcc] + _flags(src, flags) + ["-c", "-o", obj, os.path.join(CSRC, src)]))
    failed = [src for src, p in zip(SOURCES, procs) if p.wait() != 0]
    if failed:
        raise RuntimeError(f"nvcc failed on {failed}")
    subprocess.check_call([nvcc] + GENCODE + ["-shared", "-o", LIB_PATH] + objs)
    return LIB_PATH
