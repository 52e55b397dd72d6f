"""Build libegovlp_b200.so (all CUDA sources under csrc/) for sm_90a (H100) with nvcc, in-tree.

    python -m egovlp_b200.build [--force]

Objects are compiled in parallel and cached by source mtime; the shared library lands in
egovlp_b200/lib/ (git-ignored).
"""
import concurrent.futures as cf
import glob
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "build")
LIB_DIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIB_DIR, "libegovlp_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [ "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC]
# IEEE fp32 (no --use_fast_math: no approximate division / sqrt / exp, no flush-to-zero) where the reference computes in
# fp32 and the results are compared at fp32 rounding level or bit-exactly: losses, ranking metrics, EgoMCQ, AdamW, and the
# dataset video transforms (b / 255 and the normalisation are divisions, as torch's), and the BERT pooler's tanh.
IEEE_SOURCES = {"loss.cu", "loss_fused.cu", "retrieval.cu", "optim.cu", "video_transform.cu", "text_pooler.cu"}


def flags_for(src):
    return NVCC_FLAGS + ([] if os.path.basename(src) in IEEE_SOURCES else ["--use_fast_math"])


def nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; libegovlp_b200.so must be prebuilt (python -m egovlp_b200.build)")
    return exe


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)
    srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
    hdrs = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(ROOT, "include", "*.h"))
    jobs = []
    objs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s)[:-3] + ".o")
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            jobs.append([nvcc()] + flags_for(s) + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for cmd, r in ex.map(run, jobs):
                if verbose or r.returncode:
                    sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
                if r.returncode:
                    raise RuntimeError("nvcc failed for " + cmd[-3])
    if force or jobs or _stale(LIB, objs):
        cmd = [nvcc(), "-shared", "-o", LIB] + objs + ARCH
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
