"""Build libcurate_b200.so in-tree with nvcc for sm_90a (no JIT cache: the .so travels with the tree)."""

from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libcurate_b200.so"
STAMP = PKG / ".libcurate_b200.stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--use_fast_math=false",
    "-Xcompiler", "-fPIC,-O3,-fno-fast-math,-ffp-contract=off", "--expt-relaxed-constexpr",
    "-Xptxas", "-v", "-shared", "-cudart", "shared",
]  # fmt: skip
NVCC_FLAGS = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]


def sources() -> list[Path]:
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*")) + [PKG.parent / "include" / "curate_b200.h"]):
        if p.is_file():
            h.update(p.name.encode())
            h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def nvcc_path() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libcurate_b200 cannot be built (there is no CPU fallback)")


def _headers_digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + [PKG.parent / "include" / "curate_b200.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """One object per source (compiled in parallel, cached by content hash under build/), then one link."""
    from concurrent.futures import ThreadPoolExecutor

    dig = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == dig:
        return LIB
    nvcc = nvcc_path()
    objdir = PKG / "build"
    objdir.mkdir(exist_ok=True)
    hdr = _headers_digest()
    compile_flags = [f for f in NVCC_FLAGS if f not in ("-shared",)]
    logs: list[str] = []

    def compile_one(src: Path) -> Path:
        key = hashlib.sha256(src.read_bytes() + hdr.encode()).hexdigest()[:20]
        obj = objdir / f"{src.stem}.{key}.o"
        if obj.exists() and not force:
            return obj
        for old in objdir.glob(f"{src.stem}.*.o"):
            old.unlink()
        cmd = [nvcc, *compile_flags, "-x", "cu", "-c", str(src), "-o", str(obj)]
        res = subprocess.run(cmd, capture_output=True, text=True, cwd=str(CSRC))
        logs.append(" ".join(cmd) + "\n" + res.stdout + "\n" + res.stderr)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src.name}:\n{res.stderr[-4000:]}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as tp:
        objs = list(tp.map(compile_one, sources()))
    cmd = [nvcc, "-shared", "-cudart", "shared", "-gencode", "arch=compute_90a,code=sm_90a", *[str(o) for o in objs], "-o", str(LIB), "-ldl"]
    res = subprocess.run(cmd, capture_output=True, text=True, cwd=str(CSRC))
    logs.append(" ".join(cmd) + "\n" + res.stdout + "\n" + res.stderr)
    (PKG / "build.log").write_text("\n".join(logs))
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stderr[-4000:]}")
    if verbose:
        print("\n".join(logs))
    STAMP.write_text(dig)
    return LIB


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose=True))
