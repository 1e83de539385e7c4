"""Builds libsearcharray_b200.so in-tree with nvcc for sm_90a (H100; no GPU needed to compile)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsearcharray_b200.so")
SOURCES = ["sa_index.cu", "sa_term.cu", "sa_topk.cu", "sa_phrase.cu", "sa_span.cu", "sa_filter.cu", "sa_edismax.cu", "sa_similarity.cu", "sa_comm.cu", "sa_setops.cu", "sa_build.cu",
           "sa_view.cu", "sa_bool.cu", "sa_feature.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-fmad=false"]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


SYNTH_LIB = os.path.join(HERE, "libsa_synth.so")


def build_synth(force=False):
    """The synthetic-corpus generator (host C + pthreads; bench / test data infrastructure)."""
    src = os.path.join(CSRC, "sa_synth.c")
    if force or _newer(SYNTH_LIB, [src]):
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-pthread", "-shared", "-fPIC", "-Wall",
                               "-o", SYNTH_LIB, src, "-lm"])
    return SYNTH_LIB


def build(force=False, verbose=False):
    build_synth(force)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "searcharray_b200.h"))
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(o, [s] + headers):
            cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write(out.decode())
        if p.returncode:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    if force or procs or _newer(LIB, objs):
        cmd = [nvcc, "-shared", "-o", LIB + ".tmp"] + objs + ["-lcudart", "-ldl"]   # NCCL is dlopen'ed (sa_comm.cu)
        subprocess.check_call(cmd)
        os.replace(LIB + ".tmp", LIB)          # atomic: a concurrent reader never sees a half-written library
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
