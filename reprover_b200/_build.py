"""In-tree native build: nvcc (sm_90a) for the engine, gcc for the C oracle.

The engine library is `reprover_b200/_lib/librpx.so`; it is built from
`reprover_b200/csrc/*.cu` with

    nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 ...

nvcc cross-compiles without a GPU, so the build needs no device; the library is
a build product (git-ignored) and is rebuilt from a clean checkout.  Nothing here
falls back to another architecture or to a CPU implementation.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
REPO_ROOT = PKG_DIR.parent
CSRC = PKG_DIR / "csrc"
# RPX_LIB_VARIANT=<name> selects a side-by-side build (tuning experiments: A/B on the same GPU box)
_VARIANT = os.environ.get("RPX_LIB_VARIANT", "")
LIB_DIR = PKG_DIR / "_lib"
OBJ_DIR = LIB_DIR / ("obj_" + _VARIANT if _VARIANT else "obj")
LIB_PATH = LIB_DIR / (f"librpx_{_VARIANT}.so" if _VARIANT else "librpx.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


# extra defines for tuning experiments, e.g. RPX_NVCC_EXTRA="-DRPX_PREFETCH_KB=0"
NVCC_FLAGS += [f for f in os.environ.get("RPX_NVCC_EXTRA", "").split() if f]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the engine cannot be built (there is no fallback path)")


def _sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _deps_digest() -> str:
    """Digest of every file a translation unit may include (headers + public ABI)."""
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + [REPO_ROOT / "include" / "rpx.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _compile_one(nvcc: str, src: Path, obj: Path, log: Path) -> None:
    cmd = [nvcc, *NVCC_FLAGS, "-I", str(REPO_ROOT / "include"), "-c", str(src), "-o", str(obj)]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    log.write_text("$ " + " ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{proc.stdout}\n{proc.stderr}")


def build_engine(force: bool = False, verbose: bool = True) -> Path:
    """Compile every `.cu` under csrc/ for sm_90a and link `librpx.so` (incremental)."""
    nvcc = _nvcc()
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    deps = _deps_digest()
    todo = []
    objs = []
    for src in _sources():
        obj = OBJ_DIR / (src.stem + ".o")
        stamp = OBJ_DIR / (src.stem + ".stamp")
        want = hashlib.sha256(src.read_bytes() + deps.encode()).hexdigest()
        objs.append(obj)
        if force or not obj.exists() or not stamp.exists() or stamp.read_text() != want:
            todo.append((src, obj, stamp, want))
    if todo:
        if verbose:
            print(f"[rpx build] nvcc sm_90a: {', '.join(s.name for s, *_ in todo)}", file=sys.stderr)
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            futs = [ex.submit(_compile_one, nvcc, s, o, OBJ_DIR / (s.stem + ".log")) for s, o, _, _ in todo]
            for f in futs:
                f.result()
        for _, _, stamp, want in todo:
            stamp.write_text(want)
    if todo or not LIB_PATH.exists():
        cmd = [nvcc, "-shared", "-o", str(LIB_PATH), *map(str, objs),
               "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
               "-Xlinker", "--no-undefined"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError(f"link failed:\n{proc.stdout}\n{proc.stderr}")
        if verbose:
            print(f"[rpx build] linked {LIB_PATH}", file=sys.stderr)
    return LIB_PATH


# --------------------------------------------------------------------------- oracle (test infra)
ORACLE_DIR = REPO_ROOT / "oracle"
ORACLE_LIB = ORACLE_DIR / "_build" / "librpx_oracle.so"


def build_oracle(force: bool = False, verbose: bool = True) -> Path:
    """gcc build of the C oracle (`oracle/rpx_oracle.c`).  Test infrastructure only."""
    src = ORACLE_DIR / "rpx_oracle.c"
    ORACLE_LIB.parent.mkdir(parents=True, exist_ok=True)
    if not force and ORACLE_LIB.exists() and ORACLE_LIB.stat().st_mtime >= src.stat().st_mtime:
        return ORACLE_LIB
    cmd = ["gcc", "-O2", "-std=c11", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off",
           "-o", str(ORACLE_LIB), str(src), "-lm"]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"oracle build failed:\n{proc.stdout}\n{proc.stderr}")
    if verbose:
        print(f"[rpx build] built {ORACLE_LIB}", file=sys.stderr)
    return ORACLE_LIB


if __name__ == "__main__":
    build_engine(force="--force" in sys.argv)
    if (ORACLE_DIR / "rpx_oracle.c").exists():
        build_oracle(force="--force" in sys.argv)
