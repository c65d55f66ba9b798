"""In-tree build of the xb200 C-ABI shared library (nvcc, sm_90a only: H100).

    python -m xuance_b200.build [--force]

Produces xuance_b200/libxb200.so next to this file (git-ignored, rebuilt when a source or a flag changes).  No torch
headers are involved: the library is plain CUDA runtime + extern "C"."""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libxb200.so")
STAMP = os.path.join(HERE, ".libxb200.stamp")
SOURCES = ["api.cu", "rollout.cu", "losses.cu", "per_tree.cu", "optim.cu", "sac.cu", "ddpg.cu", "dist_dqn.cu", "ppg.cu", "gru.cu", "lstm.cu", "qmix_mix.cu", "qmix_tc.cu", "wqmix.cu", "dcg.cu", "qtran.cu", "vdac.cu", "coma.cu", "act.cu", "conv_tc.cu", "obs_planes.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--use_fast_math=false", "-ftz=false", "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v",
              "--expt-relaxed-constexpr", "--expt-extended-lambda"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest(files):
    h = hashlib.sha256()
    for f in files:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def build(force=False, verbose=False):
    srcs = sources()
    deps = srcs + [os.path.join(CSRC, "xb_common.cuh"), os.path.join(HERE, "..", "include", "xb200.h")]
    deps += [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")) and f != "xb_common.cuh"]
    dig = _digest(sorted(set(deps)))
    if not force and os.path.exists(OUT) and os.path.exists(STAMP) and open(STAMP).read().strip() == dig:
        return OUT
    flags = [f for f in NVCC_FLAGS if f != "--use_fast_math=false"]
    cmd = [_nvcc()] + flags + ["-o", OUT] + srcs
    res = subprocess.run(cmd, capture_output=True, text=True)
    log = res.stdout + res.stderr
    with open(os.path.join(HERE, "build.log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + log)
    if res.returncode != 0:
        sys.stderr.write(log)
        raise RuntimeError("nvcc failed building libxb200.so")
    if verbose:
        print(log)
    with open(STAMP, "w") as fh:
        fh.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
