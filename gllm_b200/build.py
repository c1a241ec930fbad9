"""In-tree build of the sm_90a kernel library (`gllm_b200/_C/libgllm_b200.so`).

Plain `nvcc` -> one shared object with a C ABI (loaded through ctypes in
`gllm_b200.ops.lib`). No torch headers are needed, so a full rebuild takes
seconds and cross-compiles on a GPU-less box.

    python -m gllm_b200.build [--force] [--verbose]
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
OUT_DIR = os.path.join(ROOT, "_C")
LIB_PATH = os.path.join(OUT_DIR, "libgllm_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--use_fast_math",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]


def _sources() -> list[str]:
    out = []
    for d, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith(".cu") or f.endswith(".cpp"):
                out.append(os.path.join(d, f))
    return sorted(out)


def _headers() -> list[str]:
    out = []
    for d, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".h", ".cuh", ".hpp")):
                out.append(os.path.join(d, f))
    return sorted(out)


def _digest(paths: list[str]) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    for p in paths:
        h.update(p.encode())
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def nvcc_path() -> str:
    cand = os.environ.get("NVCC", "")
    if cand and os.path.exists(cand):
        return cand
    for c in ("/usr/local/cuda/bin/nvcc",):
        if os.path.exists(c):
            return c
    return "nvcc"


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    srcs = _sources()
    hdr_digest = _digest(_headers())
    stamp_path = os.path.join(OUT_DIR, "build.stamp")
    objs = []
    todo = []
    for s in srcs:
        rel = os.path.relpath(s, CSRC).replace(os.sep, "_")
        obj = os.path.join(OUT_DIR, rel + ".o")
        dig = _digest([s]) + hdr_digest
        digf = obj + ".sha"
        objs.append(obj)
        old = open(digf).read() if os.path.exists(digf) else ""
        if force or old != dig or not os.path.exists(obj):
            todo.append((s, obj, dig, digf))

    def compile_one(item):
        s, obj, dig, digf = item
        cmd = [nvcc_path(), *NVCC_FLAGS, "-I", CSRC, "-c", s, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas")
            cmd.insert(2, "-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(r.stderr)
        with open(digf, "w") as f:
            f.write(dig)
        return s

    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            for s in ex.map(compile_one, todo):
                print(f"[gllm_b200.build] compiled {os.path.relpath(s, ROOT)}")
    if todo or not os.path.exists(LIB_PATH):
        cmd = [nvcc_path(), "-shared", "-o", LIB_PATH, *objs, "-lpthread"]  # static cudart (nvcc default)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
        print(f"[gllm_b200.build] linked {LIB_PATH}")
        with open(stamp_path, "w") as f:
            f.write(hdr_digest)
    return LIB_PATH


def main():
    build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)


if __name__ == "__main__":
    main()
