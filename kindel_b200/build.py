"""In-tree build of libkindel_b200.so (H100, sm_90a) and of the oracle's C restatement.

`python -m kindel_b200.build` (or `__graft_entry__.build()`) compiles

    kindel_b200/csrc/api.cu (+ the kernel files it includes) + bam_host.cpp (links zlib)
        -> kindel_b200/_lib/libkindel_b200.so          nvcc, -gencode arch=compute_90a,code=sm_90a
    oracle/kindel_oracle.c -> oracle/_build/libkindel_oracle.so   gcc (test infrastructure)
    oracle/kindel_qoracle.c -> oracle/_build/libkindel_qoracle.so gcc (test infrastructure: the base-quality filter)
    oracle/kindel_ioracle.c, kindel_fqoracle.c -> oracle/_build/  gcc (test infrastructure: the IUPAC vote, the
                                                                  per-base consensus qualities)

Both artefacts are git-ignored.  A rebuild is skipped when the artefact is newer than every source and than
this file (which holds the compiler flags).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kindel_b200", "csrc")
LIB_DIR = os.path.join(ROOT, "kindel_b200", "_lib")
LIB_PATH = os.path.join(LIB_DIR, "libkindel_b200.so")
ORACLE_SRC = os.path.join(ROOT, "oracle", "kindel_oracle.c")
ORACLE_DIR = os.path.join(ROOT, "oracle", "_build")
ORACLE_LIB = os.path.join(ORACLE_DIR, "libkindel_oracle.so")
QORACLE_SRC = os.path.join(ROOT, "oracle", "kindel_qoracle.c")
QORACLE_LIB = os.path.join(ORACLE_DIR, "libkindel_qoracle.so")
IORACLE_SRC = os.path.join(ROOT, "oracle", "kindel_ioracle.c")
IORACLE_LIB = os.path.join(ORACLE_DIR, "libkindel_ioracle.so")
FQORACLE_SRC = os.path.join(ROOT, "oracle", "kindel_fqoracle.c")
FQORACLE_LIB = os.path.join(ORACLE_DIR, "libkindel_fqoracle.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-fvisibility=default",
    "-Xptxas", "-v",
    "-shared", "-cudart", "static",
]


def _newer(target: str, sources: list[str]) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; the CUDA engine cannot be built")
    return exe


def build_engine(force: bool = False, verbose: bool = False) -> str:
    sources = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    sources += [os.path.join(ROOT, "include", "kindel_b200.h"), os.path.abspath(__file__)]
    if not force and _newer(LIB_PATH, sources):
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    cmd = [_nvcc(), *NVCC_FLAGS, "-I", os.path.join(ROOT, "include"),
           os.path.join(CSRC, "api.cu"), os.path.join(CSRC, "bam_host.cpp"), "-lz", "-o", LIB_PATH]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(LIB_DIR, "build.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + log)
    if verbose:
        print(log, file=sys.stderr)
    return LIB_PATH


def build_oracle(force: bool = False) -> str:
    """The C checkers (the pileup restatement, its base-quality-masking variant, the IUPAC vote and the consensus
    qualities); returns the first's path."""
    for src, lib in ((ORACLE_SRC, ORACLE_LIB), (QORACLE_SRC, QORACLE_LIB), (IORACLE_SRC, IORACLE_LIB),
                     (FQORACLE_SRC, FQORACLE_LIB)):
        if not force and _newer(lib, [src, os.path.abspath(__file__)]):
            continue
        os.makedirs(ORACLE_DIR, exist_ok=True)
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-std=c11", "-Wall", src, "-o", lib]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("gcc failed building the oracle:\n" + res.stdout + res.stderr)
    return ORACLE_LIB


def main(argv=None) -> int:
    argv = sys.argv[1:] if argv is None else argv
    force = "--force" in argv
    print(build_engine(force=force, verbose="-v" in argv))
    print(build_oracle(force=force))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
