"""Builds libtrinity_b200.so (sm_90a CUDA kernels + host C++ + C ABI) in-tree with nvcc.

Run as `python -m trinity_b200.build` or through `__graft_entry__.build()`.  The shared object and the
object files under build/ are git-ignored.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIB = ROOT / "libtrinity_b200.so"
OBJ = ROOT / "build"

CU_SOURCES = ["kernels.cu", "engine.cu"]
CXX_SOURCES = ["codecs.cpp", "host_api.cpp", "planner.cpp", "segment.cpp"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-pthread"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found: trinity_b200 has no CPU fallback and cannot be built without the CUDA toolkit")


def _stale() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = list(CSRC.glob("*")) + [ROOT.parent / "include" / "trinity_b200.h", Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def build_native(force: bool = False, verbose: bool = False) -> Path:
    if not force and not _stale():
        return LIB
    nvcc = _nvcc()
    OBJ.mkdir(exist_ok=True)
    objs = []
    procs = []
    for src in CU_SOURCES:
        o = OBJ / (src + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-Xptxas", "-v", "-c", str(CSRC / src), "-o", str(o)]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    for src in CXX_SOURCES:
        o = OBJ / (src + ".o")
        cmd = ["g++", *CXX_FLAGS, "-I/usr/local/cuda/include", "-c", str(CSRC / src), "-o", str(o)]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src}\n{out}")
        failed |= p.returncode != 0
    (OBJ / "build.log").write_text("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("trinity_b200 native build failed (see above)")
    if verbose:
        print("\n".join(log))
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-Xcompiler", "-pthread", "-lpthread"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("trinity_b200 link failed")
    return LIB


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose=True))
