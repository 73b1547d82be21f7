"""ygz_slam_b200 -- H100-native (sm_90a) implementation of the ygz-slam per-frame tracking + local-BA
hot path behind the C ABI of include/ygz_b200.h.

The compute lives in csrc/ (hand-written CUDA, built in-tree into libygz_b200.so by build.py); this
package only holds the ctypes binding used by the tests and the benchmark, the seeded synthetic input
generators, and the C++ shim classes (host/) that keep the reference's call surface.
There is no CPU fallback: loading the library or creating a context fails loudly without it / an H100 (sm_90).
"""
from .capi import Context, Frames, YgzbError, load_library, lib_path, undistort_map  # noqa: F401
