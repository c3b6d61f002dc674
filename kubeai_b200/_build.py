"""Build libb200engine.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

The shared library is the product: a C-ABI engine (include/b200engine.h) with no Python or torch
dependency.  Python only loads it through ctypes (kubeai_b200/_lib.py).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIB = ROOT / "lib" / "libb200engine.so"
OBJ = ROOT / "lib" / "obj"

SOURCES = [
    "gemm_wgmma.cu",
    "attention.cu",
    "attention_wgmma.cu",
    "elementwise.cu",
    "sampling.cu",
    "penalties.cu",
    "kv_fork.cu",
    "pooling.cu",
    "abi_ops.cu",
    "engine.cu",
    "router.cc",
    "loader.cc",
    "tokenizer.cc",
    "server.cc",
    "harness.cc",
]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function",
    "-diag-suppress", "177",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(str(p).encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    srcs = [CSRC / s for s in SOURCES if (CSRC / s).exists()]
    deps = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + [ROOT.parent / "include" / "b200engine.h"] + \
        list((ROOT.parent / "cmd").glob("*.cc"))
    stamp = OBJ / "digest.txt"
    digest = _digest(srcs + deps)
    if not force and LIB.exists() and stamp.exists() and stamp.read_text() == digest:
        return LIB
    OBJ.mkdir(parents=True, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: Path) -> Path:
        obj = OBJ / (src.name + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-x", "cu", "-c", str(src), "-o", str(obj)]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    cmd = [nvcc, "-shared", "-o", str(LIB), *map(str, objs), "-lcudart", "-lpthread", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    # the two process entry points (cmd/): server and load generator, linked against the library
    bindir = ROOT / "bin"
    bindir.mkdir(exist_ok=True)
    for name in ("b200serve", "b200bench"):
        src = ROOT.parent / "cmd" / f"{name}.cc"
        if not src.exists():
            continue
        cmd = [nvcc, "-O2", "-std=c++17", "-x", "cu", str(src), "-o", str(bindir / name), "-L", str(LIB.parent),
               "-lb200engine", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../lib", "-lcudart", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"building {name} failed:\n{r.stdout}\n{r.stderr}")
    stamp.write_text(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
