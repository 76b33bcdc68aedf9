"""Build of the in-tree CUDA library (sm_90a only, no multi-arch fallbacks)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libknowhere_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-fopenmp,-O3,-mavx2,-mfma", "-shared",
]


# the translation units of the library, in link order: every build of it (also scripts/filter_stalls.py) compiles these.
# kb2_muvera_proj.cpp is a host unit of its own, compiled without FMA contraction (see its header).
UNITS = [os.path.join(CSRC, "kb2_capi.cu"), os.path.join(CSRC, "kb2_muvera_proj.cpp")]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".h", ".cpp")))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    hdr = os.path.join(os.path.dirname(HERE), "include", "knowhere_b200.h")
    return any(os.path.getmtime(s) > t for s in sources() + [hdr])


def build(force=False, verbose=False):
    """nvcc -> knowhere_b200/libknowhere_b200.so (in-tree, so it travels to the GPU box)."""
    if not force and not needs_build():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc] + NVCC_FLAGS + ["-o", LIB] + UNITS + ["-lgomp", "-ldl"]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return LIB
