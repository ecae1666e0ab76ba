"""Build libpadel_b200.so (hand-written sm_90a CUDA + C ABI) in-tree with nvcc.

The library is torch-free: plain `nvcc -gencode arch=compute_90a,code=sm_90a` on csrc/*.cu.  The built .so and the
object directory are git-ignored build products; the build is skipped when sources and flags are unchanged.

The conv kernels (csrc/conv_*.cu) are compiled with `-Xptxas -v`; the report is kept as build/<stem>.ptxas.txt and
`ptxas_problems()` lists what would make a conv kernel slow without any run-time sign: wgmma serialisation warnings
(C7510 / C7511, the wgmma pipeline gives up for lack of registers) and register spills.
"""
from __future__ import annotations

import hashlib
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = HERE / "libpadel_b200.so"
OBJ = HERE / "build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
]
# translation units whose ptxas report is kept and checked
PTXAS_REPORT_GLOB = "conv_*.cu"


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(PTXAS_REPORT_GLOB.encode())
    return h.hexdigest()


def sources():
    return sorted(CSRC.glob("*.cu"))


def build_lib(force: bool = False, verbose: bool = False) -> Path:
    srcs = sources()
    deps = srcs + sorted(CSRC.glob("*.h")) + sorted(CSRC.glob("*.cuh")) + [HERE.parent / "include" / "padel_b200.h",
                                                                          CSRC / "exports.map"]
    stamp = OBJ / "stamp.txt"
    dig = _digest(deps)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == dig:
        return LIB
    OBJ.mkdir(exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: Path) -> Path:
        obj = OBJ / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
        report = src.match(PTXAS_REPORT_GLOB)
        if verbose or report:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        if report:
            (OBJ / (src.stem + ".ptxas.txt")).write_text(r.stderr)
        if verbose:
            print(r.stderr, file=sys.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-cudart", "static",
           "-Xlinker", f"--version-script={CSRC / 'exports.map'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(dig)
    return LIB


def ptxas_problems(obj_dir: Path = OBJ) -> list[str]:
    """Every conv_*_kernel instantiation whose wgmmas ptxas serialised (C7510 / C7511) or that spills registers, from
    the ptxas reports of the last build.  Raises if a report is missing."""
    problems = []
    for src in sorted(CSRC.glob(PTXAS_REPORT_GLOB)):
        rep = obj_dir / (src.stem + ".ptxas.txt")
        if not rep.exists():
            raise RuntimeError(f"{rep} missing: build the library first")
        func = None
        for line in rep.read_text().splitlines():
            m = re.search(r"Function properties for (\S+)", line)
            if m:
                func = m.group(1)
                continue
            m = re.search(r"\((C751[01])\).*function '([^']+)'", line)
            if m and "conv_" in m.group(2):
                problems.append(f"{src.name}: {m.group(1)} in {m.group(2)}")
                continue
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m and func and "conv_" in func and (int(m.group(1)) or int(m.group(2))):
                problems.append(f"{src.name}: {m.group(1)} bytes spill stores, {m.group(2)} bytes spill loads in {func}")
    return problems


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
