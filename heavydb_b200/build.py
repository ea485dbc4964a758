"""Builds the C-ABI shared library in-tree: heavydb_b200/libb2q.so (sm_90a, H100, only).

    python -m heavydb_b200.build [--force] [-v]

Every translation unit is compiled on its own (nvcc cross-compiles without a GPU), in parallel, into
heavydb_b200/_obj/<unit>-<hash>.o where <hash> covers the unit's source, every header of csrc/ and include/, and the
flags — so an edit recompiles only what it touches — and the objects are linked into libb2q.so.  Next to the library,
libb2q.so.srchash records the hash of ALL sources it was linked from: `needs_build()` compares hashes, not mtimes, so a
stale binary is never reused silently.  The .so and the objects are git-ignored but the .so travels to the GPU box with
the repo snapshot.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(HERE, "..", "include")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libb2q.so")
HASHFILE = LIB + ".srchash"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("CXX", "g++")
CUDA_INC = os.path.join(os.path.dirname(os.path.dirname(NVCC)), "include")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "-Xptxas", "-v"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-pthread", "-I" + CUDA_INC]

# (unit name, source file, extra defines).  scan_inst.cu holds the b2q_k_scan instantiations of one
# (join level, table-mode group); nine units so that they compile in parallel.
UNITS = [(f"scan_j{j}_g{g}", "scan_inst.cu", [f"-DB2Q_SCAN_JOIN={j}", f"-DB2Q_SCAN_GROUP={g}"]) for j in range(3) for g in range(3)]
UNITS += [("kernels", "kernels.cu", []), ("sort", "sort.cu", []), ("radix_agg", "radix_agg.cu", []), ("columnar", "columnar.cu", []), ("project", "project.cu", []),
          ("executor", "executor.cpp", []), ("multi", "multi.cpp", []), ("planner", "planner.cpp", [])]


def _headers():
    hs = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".h", ".cuh", ".hpp"))]
    hs += [os.path.join(INCLUDE, f) for f in sorted(os.listdir(INCLUDE)) if f.endswith(".h")]
    return hs


def _digest(paths, extra=()):
    h = hashlib.sha256()
    for p in paths:
        h.update(os.path.basename(p).encode())
        with open(p, "rb") as f:
            h.update(f.read())
    for e in extra:
        h.update(str(e).encode())
    return h.hexdigest()[:16]


def _units():
    return [u for u in UNITS if os.path.exists(os.path.join(CSRC, u[1]))]


def source_hash() -> str:
    srcs = sorted({os.path.join(CSRC, u[1]) for u in _units()})
    return _digest(srcs + _headers(), NVCC_FLAGS + CXX_FLAGS + [repr(_units())])


def needs_build() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(HASHFILE):
        return True
    return open(HASHFILE).read().strip() != source_hash()


def _compile(unit, log):
    name, src, defs = unit
    path = os.path.join(CSRC, src)
    cuda = src.endswith(".cu")
    flags = NVCC_FLAGS if cuda else CXX_FLAGS
    obj = os.path.join(OBJ, f"{name}-{_digest([path] + _headers(), flags + defs)}.o")
    if os.path.exists(obj):
        return obj, ""
    for old in os.listdir(OBJ):
        if old.startswith(name + "-") and old.endswith(".o"):
            os.remove(os.path.join(OBJ, old))
    cmd = ([NVCC] + NVCC_FLAGS + defs + ["-c", "-o", obj, path]) if cuda else ([CXX] + CXX_FLAGS + defs + ["-c", "-o", obj, path])
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        if os.path.exists(obj):
            os.remove(obj)
        raise RuntimeError(f"compiling {name} failed:\n{r.stdout}{r.stderr}")
    return obj, f"==== {name} ====\n{r.stderr}"


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for old in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, old))
    units = _units()
    with ThreadPoolExecutor(max_workers=max(1, min(len(units), os.cpu_count() or 1))) as pool:
        results = list(pool.map(lambda u: _compile(u, None), units))
    objs = [o for o, _ in results]
    logs = "".join(l for _, l in results)
    r = subprocess.run([NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-ldl", "-lpthread"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("linking libb2q.so failed")
    if logs:   # ptxas -v (registers, spills) of the units that were recompiled
        with open(os.path.join(HERE, "build_ptxas.log"), "a" if not force else "w") as f:
            f.write(logs)
    if verbose:
        sys.stderr.write(logs)
    with open(HASHFILE, "w") as f:
        f.write(source_hash() + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
