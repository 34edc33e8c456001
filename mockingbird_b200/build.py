"""In-tree build of libmockingbird_b200.so (nvcc, sm_90a only).

The shared library is the product's compute path; there is no CPU fallback.  The built .so is
git-ignored but travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libmockingbird_b200.so"
STAMP = PKG_DIR / ".libmockingbird_b200.hash"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-fmad=false",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-O3", "-shared", "-lpthread",
]


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cpp"))


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")) + list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh"))
                    + [PKG_DIR.parent / "include" / "mockingbird_b200.h", PKG_DIR.parent / "include" / "mb_wavernn_math.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    return LIB_PATH.is_file() and STAMP.is_file() and STAMP.read_text().strip() == _digest()


def find_nvcc() -> str | None:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.isfile(cand) else None


def _obj_digest(src: Path, headers_digest: str) -> str:
    h = hashlib.sha256()
    h.update(src.read_bytes())
    h.update(headers_digest.encode())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA / C++ source into one shared library (objects are cached per source under
    csrc/.obj and recompiled only when the source, any header or the flags changed).  Raises on failure."""
    if not force and is_fresh():
        return LIB_PATH
    nvcc = find_nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libmockingbird_b200.so")
    from concurrent.futures import ThreadPoolExecutor

    objdir = CSRC / ".obj"
    objdir.mkdir(exist_ok=True)
    hd = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + [PKG_DIR.parent / "include" / "mockingbird_b200.h",
                                                                           PKG_DIR.parent / "include" / "mb_wavernn_math.h"]):
        if p.is_file():
            hd.update(p.name.encode())
            hd.update(p.read_bytes())
    headers_digest = hd.hexdigest()
    cflags = [f for f in NVCC_FLAGS if f not in ("-shared", "-lpthread")]

    def compile_one(src: Path):
        obj = objdir / (src.name + ".o")
        stamp = objdir / (src.name + ".hash")
        dig = _obj_digest(src, headers_digest)
        if obj.is_file() and stamp.is_file() and stamp.read_text() == dig:
            return obj, None
        cmd = [nvcc, *cflags, "-c", "-o", str(obj), str(src)]
        if verbose:
            print(" ".join(cmd))
        proc = subprocess.run(cmd, cwd=str(CSRC), capture_output=True, text=True)
        if proc.returncode != 0:
            return obj, f"{src.name}:\n{proc.stdout}\n{proc.stderr}"
        stamp.write_text(dig)
        return obj, None

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 4)) as ex:
        results = list(ex.map(compile_one, sources()))
    errs = [e for _, e in results if e]
    if errs:
        raise RuntimeError("nvcc failed:\n" + "\n".join(errs))
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(LIB_PATH), *[str(o) for o, _ in results],
           "-lpthread"]
    proc = subprocess.run(cmd, cwd=str(CSRC), capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"link failed:\n{proc.stdout}\n{proc.stderr}")
    STAMP.write_text(_digest())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force=True, verbose=True))
