"""Builds ``libdotaclient_b200.so`` (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

``python -m dotaclient_b200.build`` or ``__graft_entry__.build()``.  The library links the static
CUDA runtime only -- no torch, no Python -- so the same .so serves ctypes, cgo, JNI or any other FFI.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB_PATH = os.path.join(HERE, "libdotaclient_b200.so")
ARCH = "arch=compute_90a,code=sm_90a"       # wgmma and the sm_90a feature set: H100 only
SOURCES = ["capi.cu", "gae_scan.cu", "vtrace_scan.cu", "upgo_scan.cu", "gather.cu", "ppo_loss.cu", "grad_finish.cu", "rnn_seq.cu", "gemm_tf32x3.cu", "encoder.cu", "actor.cu",
           "value_norm.cu", "state_refresh.cu", "value_heads.cu", "target_rows.cu"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compiles every .cu under csrc/ to an object and links the shared library.  Returns its path."""
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(ROOT, "include", "dotaclient_b200.h"))
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    common = ["-gencode", ARCH, "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include"), "-I", CSRC]
    if verbose:
        common += ["-Xptxas", "-v"]
    objs, procs = [], []
    for s in srcs:
        o = os.path.join(objdir, os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            procs.append((s, subprocess.Popen([nvcc] + common + ["-c", s, "-o", o],
                                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("[nvcc %s]\n%s\n" % (os.path.basename(s), out))
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(LIB_PATH, objs):
        subprocess.check_call([nvcc, "-shared", "-gencode", ARCH, "-o", LIB_PATH] + objs)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
