"""Build liblseg_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

The library is a single translation unit (csrc/lseg_b200.cu) linked against the static CUDA runtime
only; the driver API entry point it needs (cuTensorMapEncodeTiled) is resolved at run time, so the
.so loads on machines without libcuda (the C-ABI export test relies on that).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "liblseg_b200.so")
SOURCES = ["lseg_b200.cu"]
HEADERS = ["common.cuh", "gemm_tc.cuh", "mhsa.cuh", "attn_probs.cuh", "text_attn.cuh", "p2p.cuh", "evaluator.cuh", "segstats.cuh", "xent.cuh", "elementwise.cuh", "embed.cuh", "engine.cuh"]


def nvcc_path():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS]
    deps.append(os.path.join(HERE, "..", "include", "lseg_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile into a temporary file and rename it over the library (atomic: a peer process that dlopens the path sees
    either the old or the new file, never a partial one), under an exclusive file lock so that N torchrun ranks finding
    a stale library build it once, not N times into the same path."""
    import fcntl
    if not force and not needs_build():
        return LIB
    lock_path = LIB + ".lock"
    with open(lock_path, "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not needs_build():  # a peer built it while we waited
                return LIB
            tmp = f"{LIB}.tmp{os.getpid()}"
            cmd = [
                nvcc_path(),
                "-gencode", "arch=compute_90a,code=sm_90a",
                "-O3", "-std=c++17", "-lineinfo",
                "-shared", "-Xcompiler", "-fPIC",
                "-cudart", "static",
                "-o", tmp,
            ]
            if verbose:
                cmd += ["-Xptxas", "-v"]
            cmd += [os.path.join(CSRC, s) for s in SOURCES]
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                sys.stderr.write(res.stdout + res.stderr)
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc failed building liblseg_b200.so")
            if verbose:
                sys.stderr.write(res.stdout + res.stderr)
            os.replace(tmp, LIB)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
