"""Build the sm_90a (H100) shared library IN-TREE (racon_gpu_b200/libb200poa.so).

nvcc cross-compiles without a GPU; the built .so is git-ignored.  `python -m racon_gpu_b200.build` or __graft_entry__.build().
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200poa.so")
SOURCES = ["b200poa.cu", "b200aln.cu", "host/cuda_batch.cpp", "host/cuda_polisher.cpp", "host/overlap_polisher.cpp"]
HEADERS = ["poa_core.cuh", "poa_fill.cuh", "poa_simt.cuh", "cuda_buffers.hpp", "host/b200_window.hpp", "host/cuda_batch.hpp",
           "host/cuda_polisher.hpp", "host/overlap_polisher.hpp", "host/b200poa_batch.hpp", "host/window_arena.hpp", "../../include/b200poa.h",
           "aln_core.cuh", "aln_layout.cuh", "layer_cut.cuh", "host/aln_levels.hpp", "host/aln_admission.hpp",
           "host/overlap_units.hpp", "host/b200aln_aligner.hpp", "../../include/b200aln.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wextra,-pthread", "-shared", "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the POA engine has no CPU fallback")


#: test build: every DP fill hashed per sequence (poa_core.cuh POA_FILL_DIGEST, b200poa_debug_fill_digest), so that the
#: CUDA fill can be compared with its scalar twin in tests/emu, and every Hirschberg split of the overlap aligner logged
#: with hashes of its middle columns (aln_core.cuh ALN_SPLIT_DIGEST, b200aln_debug_split_log), and every alignment the
#: POA traceback adds to a graph hashed per sequence (poa_core.cuh POA_ALN_DIGEST, b200poa_debug_aln_digest), and the
#: graph after every read, every subgraph and the consensus scores hashed (poa_core.cuh POA_GRAPH_DIGEST,
#: b200poa_debug_graph_digest), and every leaf of the overlap aligner logged with its end score, a hash of its operations
#: and the walk's counters (aln_core.cuh ALN_LEAF_DIGEST, b200aln_debug_leaf_log).  Same sources and flags as the
#: product plus these defines.
DIGEST_LIB = os.path.join(HERE, "variants", "libb200poa_digest.so")
DIGEST_FLAGS = ["-DPOA_FILL_DIGEST=1", "-DALN_SPLIT_DIGEST=1", "-DPOA_ALN_DIGEST=1", "-DPOA_GRAPH_DIGEST=1",
                "-DALN_LEAF_DIGEST=1"]


def needs_build(lib: str = LIB) -> bool:
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    for f in SOURCES + HEADERS:
        path = os.path.join(CSRC, f)
        if os.path.exists(path) and os.path.getmtime(path) > t:
            return True
    return False


def build(force: bool = False, verbose: bool = False, digest: bool = False) -> str:
    """Build the product library, or with digest=True the test build DIGEST_LIB."""
    lib, extra = (DIGEST_LIB, DIGEST_FLAGS) if digest else (LIB, [])
    if not force and not needs_build(lib):
        return lib
    os.makedirs(os.path.dirname(lib), exist_ok=True)
    srcs = [os.path.join(CSRC, f) for f in SOURCES if os.path.exists(os.path.join(CSRC, f))]
    cmd = [_nvcc(), *NVCC_FLAGS, *extra, "-x", "cu", "-I", os.path.join(HERE, "..", "include"), "-I", CSRC,
           "-o", lib, *srcs]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "build.log") if not digest else lib[:-3] + ".build.log", "w") as fh:
        fh.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        sys.stderr.write(log)
        raise RuntimeError(f"nvcc failed building {os.path.basename(lib)}")
    if verbose:
        print(log)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, digest="--digest" in sys.argv))
