"""Build libjkb200.so in-tree with nvcc for sm_90a (H100; no JIT cache, the .so travels with the repo).

    python -m jukebox_b200.build [--force]
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libjkb200.so")
STAMP = os.path.join(HERE, ".libjkb200.stamp")
SOURCES = ["api.cu", "decode_engine.cu", "f32_grad.cu", "f32_path.cu", "prefill.cu", "prefill_gemm.cu", "sampling.cu", "score.cu", "select.cu", "stft_loss.cu", "vqvae_kernels.cu", "vqvae_t5.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--shared", "-Xcompiler", "-fPIC", 
              "-Xcompiler", "-Wno-unused-function", "--expt-relaxed-constexpr", "-rdc=false"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest():
    h = hashlib.sha256()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    files.append(os.path.join(os.path.dirname(HERE), "include", "jkb200.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
          [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed building libjkb200.so")
    if verbose:
        sys.stderr.write(res.stderr)
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
