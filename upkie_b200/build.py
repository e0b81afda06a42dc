# SPDX-License-Identifier: Apache-2.0
"""In-tree build of ``libupkie_b200.so`` with nvcc for sm_90a (H100)."""

import os
import subprocess
from typing import NamedTuple

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libupkie_b200.so")

# the step-kernel families, numbered as in csrc/step_family.h
(FAM_PLAIN, FAM_EXTRAS, FAM_LIMITS, FAM_SPINE, FAM_BODY, FAM_TABLE, FAM_PUSH, FAM_BODY_PUSH, FAM_DELAY,
 FAM_BODY_DELAY, FAM_SENSE) = range(11)


class StepUnit(NamedTuple):
    """A translation unit of step kernels: csrc/step_unit.cu compiled for one TILE and one or two families"""
    name: str        # object name
    tile: int        # 0 device buffers, 1 host-buffer tiles, 2 in-kernel rollout transport
    families: tuple  # FAM_* of csrc/step_family.h
    body: int        # UPKIE_BODY_CONTACTS_BUILD: 1 exactly when the families have the `body` trait

    def flags(self) -> list:
        return [f"-DUPKIE_STEP_TILE={self.tile}", f"-DUPKIE_BODY_CONTACTS_BUILD={self.body}"] + [
            f"-DUPKIE_STEP_FAMILY{k}={f}" for k, f in enumerate(self.families)]


# The objects of the library in link order, compiled in parallel: the handle-side units by source file, and one step
# unit per TILE and family (plain and extras share one), whose (TILE, family) pairs are those of step_instantiated
# (csrc/step_family.h). The order places the kernels' code: keep it.
UNITS = [
    "upkie_b200.cu",
    StepUnit("step_device", 0, (FAM_PLAIN, FAM_EXTRAS), 0),
    StepUnit("step_host", 1, (FAM_PLAIN, FAM_EXTRAS), 0),
    StepUnit("step_multicast", 2, (FAM_PLAIN, FAM_EXTRAS), 0),
    StepUnit("step_device_limits", 0, (FAM_LIMITS,), 0),
    StepUnit("step_host_limits", 1, (FAM_LIMITS,), 0),
    StepUnit("step_multicast_limits", 2, (FAM_LIMITS,), 0),
    StepUnit("step_device_spine", 0, (FAM_SPINE,), 1),
    StepUnit("step_host_spine", 1, (FAM_SPINE,), 1),
    StepUnit("step_device_body", 0, (FAM_BODY,), 1),
    StepUnit("step_host_body", 1, (FAM_BODY,), 1),
    StepUnit("step_device_table", 0, (FAM_TABLE,), 0),
    StepUnit("step_host_table", 1, (FAM_TABLE,), 0),
    "base_velocity.cu",
    StepUnit("step_device_push", 0, (FAM_PUSH,), 0),
    StepUnit("step_host_push", 1, (FAM_PUSH,), 0),
    StepUnit("step_device_body_push", 0, (FAM_BODY_PUSH,), 1),
    StepUnit("step_host_body_push", 1, (FAM_BODY_PUSH,), 1),
    StepUnit("step_device_delay", 0, (FAM_DELAY,), 0),
    StepUnit("step_host_delay", 1, (FAM_DELAY,), 0),
    StepUnit("step_device_body_delay", 0, (FAM_BODY_DELAY,), 1),
    StepUnit("step_host_body_delay", 1, (FAM_BODY_DELAY,), 1),
    StepUnit("step_device_sense", 0, (FAM_SENSE,), 0),
    StepUnit("step_host_sense", 1, (FAM_SENSE,), 0),
]
# every source and header of the library: the staleness check and the key of source_hash
DEPS = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h"))) + [
    os.path.join(_HERE, "..", "include", "upkie_b200.h")]

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


def compile_jobs(units: list) -> list:
    """(object name, source file, extra flags) of each unit"""
    return [(u.name, "step_unit.cu", u.flags()) if isinstance(u, StepUnit) else (os.path.splitext(u)[0], u, [])
            for u in units]


def source_hash() -> str:
    """sha256 (first 16 hex digits) over the CUDA sources and compile flags of the library: the key that ties a
    committed ncu sidecar (``profiles/ncu_sidecar.json``, written by ``tools/ncu_summary.py``) to the build that is
    benchmarked. Stable across rebuilds and machines, unlike a hash of the binary."""
    import hashlib

    h = hashlib.sha256()
    for d in DEPS:
        with open(d, "rb") as f:
            h.update(os.path.relpath(d, CSRC).encode() + b"\0" + f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    for name, _, flags in compile_jobs(UNITS):
        h.update(" ".join([name] + flags).encode())
    return h.hexdigest()[:16]


def _is_stale(lib: str) -> bool:
    # build.py holds the unit table
    return not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in DEPS + [__file__])


def _build(units: list, flags: list, objdir: str, lib: str, what: str) -> str:
    nvcc = os.environ.get("NVCC", "nvcc")
    os.makedirs(objdir, exist_ok=True)
    objs, procs = [], []
    for name, src, extra in compile_jobs(units):
        obj = os.path.join(objdir, name + ".o")
        objs.append(obj)
        f = [x for x in flags if x != "--use_fast_math"] if src in IEEE_SOURCES else flags
        procs.append((name, subprocess.Popen([nvcc] + f + extra + ["-c", "-o", obj, os.path.join(CSRC, src)])))
    failed = [name for name, p in procs if p.wait() != 0]
    if failed:
        raise RuntimeError(f"nvcc ({what}) failed on {failed}")
    subprocess.check_call([nvcc] + GENCODE + ["-shared", "-o", lib] + objs)
    return lib


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA library (cross-compiles without a GPU)."""
    if not force and not _is_stale(LIB_PATH):
        return LIB_PATH
    flags = NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else [])
    return _build(UNITS, flags, os.path.join(_HERE, "build"), LIB_PATH, "library")


# ---- exact-arithmetic build (test / measurement companion of the product library) ------------------------------------
# Same sources WITHOUT --use_fast_math (IEEE division / sqrt / sincos, no flush-to-zero), device-buffer kernels only
# (the step units of TILE=0 with plain, extras, extras + limits); the step dispatch reports the other families as
# cudaErrorNotSupported (step_instantiated narrows to these under UPKIE_EXACT_BUILD), and so does the flush of the
# in-kernel rollout transport. Used by tests/test_gpu_exact_mode.py and bench.py's `exact_mode` line: what the one
# shortcut of the timed kernel (fast-math) costs in accuracy and buys in time.
EXACT_LIB_PATH = os.path.join(_HERE, "libupkie_b200_exact.so")
EXACT_UNITS = [u for u in UNITS if not isinstance(u, StepUnit) or (u.tile == 0 and max(u.families) <= FAM_LIMITS)]
EXACT_FLAGS = [f for f in NVCC_FLAGS if f != "--use_fast_math"] + ["-DUPKIE_EXACT_BUILD=1"]


def build_exact(force: bool = False) -> str:
    if not force and not _is_stale(EXACT_LIB_PATH):
        return EXACT_LIB_PATH
    return _build(EXACT_UNITS, EXACT_FLAGS, os.path.join(_HERE, "build", "exact"), EXACT_LIB_PATH, "exact build")
