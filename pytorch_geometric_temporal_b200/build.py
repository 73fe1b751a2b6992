"""Build libstmp.so (sm_90a, H100) in-tree with nvcc.  `python -m pytorch_geometric_temporal_b200.build`."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "libstmp.so")
SOURCES = ["plan.cu", "spmm.cu", "dcrnn_seq.cu", "dcrnn_seq_tc.cu", "gemm_tc.cu", "cells.cu", "dcrnn_bwd.cu", "tgcn_attn.cu", "gemm_blocks.cu", "astgcn_factors.cu", "train.cu", "wgrad_tc.cu"]
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


def build(force=False, verbose=False, extra_flags=(), out=None):
    """`extra_flags` / `out`: build a VARIANT of the library (e.g. -DSTMP_X=1 into lib/libstmp_x.so) next to the product one, to A/B it on
    one GPU box through the STMP_LIB environment variable (tests/perf only; the product build takes neither)."""
    if out is not None:
        return _build_variant(list(extra_flags), out)
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


def _build_variant(flags, out):
    objdir = os.path.join(HERE, "lib", "variant_" + os.path.basename(out).replace(".so", ""))
    os.makedirs(objdir, exist_ok=True)
    procs, objs = [], []
    for s in SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        cmd = [_nvcc(), *[f for f in NVCC_FLAGS if f not in ("-Xptxas", "-v")], *flags, "-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    for s, p in procs:
        o, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{o}")
    subprocess.check_call([_nvcc(), "-shared", "-o", out, *objs, "-gencode", "arch=compute_90a,code=sm_90a"])
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
