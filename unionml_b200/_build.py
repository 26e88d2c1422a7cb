"""Build the CUDA library in-tree: unionml_b200/_lib/libuml_b200.so (sm_90a only).

nvcc cross-compiles without a GPU, so this runs in the build container and the resulting .so travels to the GPU
box with the repo snapshot.  One object per .cu (compiled in parallel), then one link.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB_DIR = PKG / "_lib"
LIB = LIB_DIR / "libuml_b200.so"
OBJ_DIR = PKG.parent / "build" / "obj"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(exe).exists():
        raise RuntimeError("nvcc not found; cannot build libuml_b200.so")
    return exe


def sources():
    return sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cpp"))  # .cpp: host-only helpers (g++ through nvcc)


def _stale(out: Path, deps) -> bool:
    if not out.exists():
        return True
    t = out.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    LIB_DIR.mkdir(parents=True, exist_ok=True)
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    headers = list(CSRC.glob("*.cuh")) + list((PKG.parent / "include").glob("*.h"))
    jobs = []
    for src in sources():
        obj = OBJ_DIR / (src.stem + ".o")
        if force or _stale(obj, [src, *headers]):
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        return r.stderr

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for log in ex.map(compile_one, jobs):
                if verbose and log:
                    print(log, file=sys.stderr)
    objs = [OBJ_DIR / (s.stem + ".o") for s in sources()]
    if force or jobs or _stale(LIB, objs):
        cmd = [nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    build_pylist(force)
    return LIB


PYLIST_SRC = PKG / "csrc_host" / "uml_pylist.c"
PYLIST_LIB = LIB_DIR / "libuml_pylist.so"


def build_pylist(force: bool = False) -> Path:
    """The CPython list helper (host glue of the `List[float]` contract; gcc, no CUDA)."""
    import sysconfig

    LIB_DIR.mkdir(parents=True, exist_ok=True)
    if force or _stale(PYLIST_LIB, [PYLIST_SRC]):
        cc = shutil.which("gcc") or shutil.which("cc")
        if cc is None:
            raise RuntimeError("gcc not found; cannot build libuml_pylist.so")
        cmd = [cc, "-O2", "-shared", "-fPIC", f"-I{sysconfig.get_paths()['include']}", str(PYLIST_SRC), "-o", str(PYLIST_LIB)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"building {PYLIST_LIB.name} failed:\n{r.stdout}\n{r.stderr}")
    return PYLIST_LIB


PROBE_SRC = PKG.parent / "tests" / "cuda" / "wgmma_accum_probe.cu"
PROBE_LIB = PKG.parent / "build" / "tests" / "libwgmma_accum_probe.so"


def build_test_probes(force: bool = False) -> Path:
    """Test-only library of tests/test_gpu_wgmma_accum.py (the product never loads it): the wgmma accumulation probe,
    compiled against the product's own wgmma.cuh."""
    PROBE_LIB.parent.mkdir(parents=True, exist_ok=True)
    if force or _stale(PROBE_LIB, [PROBE_SRC, *CSRC.glob("*.cuh")]):
        cmd = [nvcc(), *NVCC_FLAGS, "-shared", str(PROBE_SRC), "-o", str(PROBE_LIB)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {PROBE_SRC.name}:\n{r.stdout}\n{r.stderr}")
    return PROBE_LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
    print(build_pylist(force="--force" in sys.argv))
