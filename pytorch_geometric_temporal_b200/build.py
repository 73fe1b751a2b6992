"""Build libstmp.so (sm_90a, H100) in-tree with nvcc.  `python -m pytorch_geometric_temporal_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libstmp.so")
SOURCES = ["plan.cu", "spmm.cu", "dcrnn_seq.cu", "dcrnn_seq_tc.cu", "gemm_tc.cu", "cells.cu", "dcrnn_bwd.cu", "dcrnn_narrow.cu", "tgcn_attn.cu", "gemm_blocks.cu", "spatial_attention_tiled.cu", "astgcn_factors.cu", "train.cu", "wgrad_tc.cu", "gru_rows.cu", "lstm_rows.cu", "dcrnn_rows.cu", "dcrnn_narrow_rows.cu", "dcrnn_wide_rows.cu", "ggc_rows.cu", "evolvegcn_rows.cu", "mpnn_rows.cu", "agcrn.cu", "hetero_rows.cu", "gman_attention.cu", "mtgnn.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "stmp.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """To A/B two versions of the library, build each in its own checkout and point STMP_LIB (_lib.py) at one of them."""
    if not force and not needs_build():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(HERE, "lib", s.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    log = []
    for s, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {s} ====\n{out}")
        if p.returncode != 0:
            sys.stderr.write("\n".join(log))
            raise RuntimeError(f"nvcc failed on {s}")
    cmd = [_nvcc(), "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.check_call(cmd)
    with open(os.path.join(HERE, "lib", "build.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
