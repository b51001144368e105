"""Build libevk_sm90.so (and nothing else) in-tree with nvcc for sm_90a (H100).

Objects go to build/ next to this file, the library next to this file; both are git-ignored.  A stamp of the sources
and flags makes a rebuild of an unchanged tree a no-op.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libevk_sm90.so")
SOURCES = ["api.cu", "gconv.cu", "gconv_tc.cu", "conv_direct.cu", "mel.cu", "elementwise.cu", "norm_weights.cu", "attention.cu",
           "vq_loss_optim.cu", "flash.cu", "gpt_misc.cu", "gemm_tma.cu", "stft.cu", "pack_batched.cu",
           "sample.cu", "bert.cu", "conv2d.cu", "lstm.cu", "bs_roformer.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _digest():
    h = hashlib.sha256()
    for name in sorted(os.listdir(CSRC)) + ["../../include/evk.h"]:
        with open(os.path.join(CSRC, name), "rb") as f:
            h.update(name.encode()); h.update(f.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    stamp = LIB + ".stamp"
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):
            return LIB      # a machine without a toolkit: use the library built on one that has it
        raise RuntimeError("nvcc not found and no prebuilt libevk_sm90.so")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src}\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    with open(stamp, "w") as f:
        f.write(dig)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
