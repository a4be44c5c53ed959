"""Builds libvqb200.so IN-TREE with nvcc for sm_90a (H100) (no torch headers: the library has a pure C ABI).

    python -m vector_quantize_pytorch_b200.build          # build if stale
    python -m vector_quantize_pytorch_b200.build --force
"""
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libvqb200.so")
SOURCES = ["vq_assign.cu", "vq_aux.cu", "vq_ema.cu", "vq_forward.cu", "vq_peer.cu", "vq_rsimvq.cu", "vq_diveq.cu", "vq_fsq.cu", "vq_lfq.cu", "vq_fsp.cu", "vq_binmap.cu", "vq_hvq.cu", "vq_rpq.cu", "vq_lq.cu"]
HEADERS = ["ptx.cuh", "vqb_common.cuh", "code_operands.cuh", "gather_row.cuh", "epilogue.cuh", "row_io.cuh", os.path.join("..", "..", "include", "vqb200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
    "-cudart", "static",
    "-Xptxas", "-v",
]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile (if stale) under an exclusive file lock: with torchrun every rank imports the package at once."""
    import fcntl
    if not force and not is_stale():
        return LIB
    with open(os.path.join(PKG, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not is_stale():  # another process built it while we waited
                return LIB
            return _build_locked(verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(verbose):
    nvcc = find_nvcc()
    if nvcc is None:
        raise RuntimeError("vqb200: nvcc not found and libvqb200.so is missing/stale; cannot build the CUDA library")
    extra = ["-DVQB_PROFILE"] if os.environ.get("VQB_PROFILE") else []  # per-role cycle counters (vqb_debug_set_profile_buffer)
    extra += os.environ.get("VQB_NVCC_EXTRA", "").split()  # A/B experiments, e.g. -DVQB_EPI_SIMPLE
    tmp = LIB + ".tmp%d" % os.getpid()
    cmd = [nvcc] + NVCC_FLAGS + extra + ["-o", tmp] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(PKG, "build.log"), "w") as f:
        f.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        raise RuntimeError("vqb200: nvcc failed\n" + log)
    os.replace(tmp, LIB)  # atomic: a concurrently importing process never sees a half-written library
    if verbose:
        print(log)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
