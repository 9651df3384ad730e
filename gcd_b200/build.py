"""Builds gcd_b200/libgcd_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m gcd_b200.build [--bf16] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["gemm.cu", "norm.cu", "elem.cu", "attn_temporal.cu", "attn_spatial.cu", "metrics.cu", "clip.cu", "render.cu", "lpips.cu"]
OUT = os.path.join(HERE, "libgcd_b200.so")


def _stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "gcd_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, bf16=False, verbose=False):
    if not force and not _stale():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        cmd = [nvcc, "-c", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3",
               "-std=c++17", "-o", obj, os.path.join(CSRC, src)]
        if bf16:
            cmd.insert(1, "-DGCD_ACT_BF16")
        cmd[1:1] = os.environ.get("GCD_NVCC_FLAGS", "").split()
        if verbose:
            cmd += ["-Xptxas", "-v"]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {src}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([nvcc, "-shared", "-Wno-deprecated-gpu-targets", "-o", OUT] + objs + ["-lcudart_static", "-ldl", "-lrt", "-lpthread"])
    return OUT


if __name__ == "__main__":
    print(build(force=True, bf16="--bf16" in sys.argv, verbose="--verbose" in sys.argv))
