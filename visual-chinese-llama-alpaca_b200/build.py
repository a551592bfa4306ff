"""Build libvcla.so (CUDA kernels + C ABI) for sm_90a (H100) with nvcc.  In-tree output: lib/libvcla.so (git-ignored)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libvcla.so")
SOURCES = ["gemm.cu", "attention.cu", "elementwise.cu", "engine.cu", "preprocess.cu", "sampler.cu", "beam.cu", "gemm_decode.cu", "attention_tc.cu", "quant.cu"]
ARCH = "arch=compute_90a,code=sm_90a"
HEADERS = ["common.cuh", "kernels.h", "logits_chain.cuh", "preprocess_core.h", os.path.join("..", "..", "include", "vcla.h")]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    procs = []
    for s in SOURCES:
        obj = os.path.join(HERE, "lib", s.replace(".cu", ".o"))
        cmd = [nvcc, "-O3", "-std=c++17", "-gencode", ARCH, "-lineinfo",
               "-Xcompiler", "-fPIC", "-Xcompiler", "-fno-strict-aliasing",
               "-c", os.path.join(CSRC, s), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    fail = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {s} (rc {p.returncode}) ---\n{out}\n")
        fail |= p.returncode != 0
    if fail:
        raise RuntimeError("nvcc failed")
    cmd = [nvcc, "-shared", "-gencode", ARCH, "-o", LIB] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
