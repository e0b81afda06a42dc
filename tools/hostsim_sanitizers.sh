#!/bin/bash
# Runs the CPU tests that execute the kernels' per-robot code (sim_core.cuh / sim_pair.cuh / mpc_core.cuh /
# observers_core.cuh / controllers_core.cuh compiled for the host, tests/hostsim) under AddressSanitizer and
# UndefinedBehaviorSanitizer: out-of-bounds indexing in the local arrays of the solvers, uninitialised reads and
# signed overflow would show up here before they show up as a corrupted robot on the GPU.
# Usage: tools/hostsim_sanitizers.sh        (from the repository root; restores the normal libhostsim.so afterwards)
set -e
cd "$(dirname "$0")/.."
LIB=tests/hostsim/libhostsim.so
python -c "import sys; sys.path.insert(0, 'tests'); import hostsim_wrap; hostsim_wrap.build()"
cp "$LIB" /tmp/libhostsim_plain.so
g++ -O1 -g -std=c++17 -fPIC -shared -fsanitize=address,undefined -fno-omit-frame-pointer -x c++ -o "$LIB" tests/hostsim/hostsim.cpp 2>/dev/null
touch "$LIB"
trap 'cp /tmp/libhostsim_plain.so "$LIB"; touch "$LIB"' EXIT
ASAN_OPTIONS=detect_leaks=0 LD_PRELOAD="$(g++ -print-file-name=libasan.so):$(g++ -print-file-name=libubsan.so)" \
  UPKIE_HOSTSIM_CXXFLAGS="-O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer" \
  python -m pytest tests/test_kernel_arithmetic_cpu.py tests/test_controllers.py tests/test_observers.py tests/test_body_contacts.py tests/test_spine_mode.py tests/test_reset_randomization_cpu.py tests/test_push_randomization_cpu.py tests/test_step_family_cpu.py -q -m "not gpu"
