"""Build libygz_b200.so (hand-written sm_90a CUDA + the extern "C" ABI) in-tree with nvcc."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = HERE / "libygz_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function",
    "-Xptxas", "-v",
]


# per-file extra flags: the f32/f64 parity kernels must not contract a*b+c into FMA
PER_FILE_FLAGS = {"align.cu": ["-fmad=false"], "track.cu": ["-fmad=false"], "initializer.cu": ["-fmad=false"],
                  "triangulate.cu": ["-fmad=false"]}


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(exe).exists():
        raise RuntimeError("nvcc not found: libygz_b200.so cannot be built (there is no CPU fallback)")
    return exe


def sources():
    return sorted(CSRC.glob("*.cu"))


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    # build.py itself is a dependency: a change of the compiler flags must rebuild the library
    deps = (list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.inc")) + [HERE.parent / "include" / "ygz_b200.h"]
            + [Path(__file__).resolve()])
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        vo_deps = [HERE / "host" / "vo_driver.cpp", HERE / "host" / "e2e_driver.cpp", HERE / "host" / "timed_threads.h",
                   HERE.parent / "include" / "ygz_vo.h"]
        if not VO_LIB.exists() or VO_LIB.stat().st_mtime < max(d.stat().st_mtime for d in vo_deps):
            build_vo_driver()
        return LIB
    objdir = HERE / "build"
    objdir.mkdir(exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = objdir / (src.stem + ".o")
        objs.append(obj)
        cmd = [nvcc(), *NVCC_FLAGS, *PER_FILE_FLAGS.get(src.name, []), "-c", str(src), "-o", str(obj)]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src.name}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src.name}")
    (objdir / "ptxas.log").write_text("\n".join(log))
    if verbose:
        print("\n".join(log))
    cmd = [nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs)]
    subprocess.run(cmd, check=True)
    build_vo_driver()
    return LIB


VO_LIB = HERE / "libygz_vo.so"


def build_vo_driver() -> Path:
    """Host-only C++ (g++): the native callers of the C ABI -- lock-step tracking loop (host/vo_driver.cpp) and the
    end-to-end extract + match loop (host/e2e_driver.cpp)."""
    srcs = [str(HERE / "host" / "vo_driver.cpp"), str(HERE / "host" / "e2e_driver.cpp")]
    gxx = shutil.which("g++") or "g++"
    cmd = [gxx, "-std=c++20", "-O3", "-fPIC", "-shared", "-Wall", "-pthread", "-o", str(VO_LIB), *srcs, f"-L{HERE}", "-lygz_b200",
           "-Wl,-rpath,$ORIGIN"]
    subprocess.run(cmd, check=True)
    return VO_LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
    print("built", LIB)
