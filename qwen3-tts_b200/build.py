"""Build libqwen3tts_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libqwen3tts_b200.so")
SOURCES = ["ar_engine.cu", "codec_engine.cu", "codec_encoder.cu", "speaker_encoder.cu", "conv_f32.cu", "gemm_sm90.cu",
           "resample.cu", "stretch.cu", "limit.cu", "loud.cu"]
NVCC_FLAGS = ["-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-cudart", "shared", "--expt-relaxed-constexpr"]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _digest(srcs):
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for fn in sorted(os.listdir(root)):
            if fn.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, fn), "rb") as f:
                    h.update(fn.encode())
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS + srcs).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    os.makedirs(LIB_DIR, exist_ok=True)
    stamp = os.path.join(LIB_DIR, "build.stamp")
    dig = _digest(srcs)
    if not force and os.path.exists(LIB_PATH) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB_PATH
    objs = []
    for s in srcs:
        obj = os.path.join(LIB_DIR, s.replace(".cu", ".o"))
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, s), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose:
            sys.stderr.write(r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{r.stdout}\n{r.stderr}")
        objs.append(obj)
    cmd = [_nvcc(), "-shared", "-cudart", "shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
