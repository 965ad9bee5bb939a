"""Builds libmmfb200.so (sm_90a only) in-tree with nvcc.

    python -m mmf_b200.csrc.build [--force] [--verbose]

The built library lives next to the sources (git-ignored).  There is exactly one target architecture:
compute_90a / sm_90a (H100).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["capi.cu", "gemm.cu", "attention.cu", "attention_varlen.cu", "attention_causal.cu", "attention_varlen_causal.cu",
           "attention_probs.cu", "rowops.cu", "optim.cu", "ce.cu", "ot.cu", "plan.cu"]
HEADERS = ["common.cuh", "mmfb_internal.h", "../../include/mmfb200.h", "../../include/mmfb200_plan.h",
           "../../include/mmfb200_update.h"]
LIB = os.path.join(HERE, "libmmfb200.so")
STAMP = os.path.join(HERE, ".build_stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _sources():
    return [s for s in SOURCES if os.path.exists(os.path.join(HERE, s))]


def _digest():
    h = hashlib.sha256()
    for f in _sources() + HEADERS:
        with open(os.path.join(HERE, f), "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu into objects (parallel) and link the shared library. Returns its path."""
    digest = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == digest:
                return LIB
    nvcc = _nvcc()
    objs, procs = [], []
    for src in _sources():
        obj = os.path.join(HERE, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(HERE, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, out))
        elif verbose:
            sys.stderr.write(out)
        else:
            # always surface spills: they are performance bugs
            for line in out.splitlines():
                if "spill" in line and "0 bytes spill stores, 0 bytes spill loads" not in line:
                    sys.stderr.write("[%s] %s\n" % (src, line))
    if failed:
        raise RuntimeError("building libmmfb200.so failed")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("linking libmmfb200.so failed:\n" + r.stdout)
    with open(STAMP, "w") as fh:
        fh.write(digest)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
