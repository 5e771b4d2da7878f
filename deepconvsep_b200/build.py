"""Build libdcs.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m deepconvsep_b200.build [--force] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdcs.so")
SOURCES = ["api.cu", "stft.cu", "stft_reg.cu", "gemm.cu", "gemm_tc.cu", "dsd.cu", "dsd_tc.cu", "dsd_convT2_tc.cu", "dsd_dense_tc.cu", "dsd_model.cu", "sconv.cu", "sconv_tc.cu", "sconv_model.cu", "bsseval.cu",
           "wiener.cu", "score1x1.cu", "score_notes.cu", "resample.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC,-O2,-Wall", "-DDCS_BUILD"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    raise RuntimeError("nvcc not found")


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "dcs.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for s in SOURCES:
        o = os.path.join(HERE, "build", s.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    fail = False
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            sys.stderr.write("== %s ==\n%s\n" % (s, out))
        fail |= p.returncode != 0
    if fail:
        raise RuntimeError("nvcc failed")
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-o", LIB] + objs
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
