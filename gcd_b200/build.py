"""Builds gcd_b200/libgcd_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m gcd_b200.build [--bf16] [--out PATH] [--verbose]

--bf16 builds the bf16-operand variant (-DGCD_ACT_BF16). Each variant compiles its objects into a directory of its own
(build/fp16/, build/bf16/), so a bf16 library written elsewhere with --out (the tests use gcd_b200/libgcd_b200_bf16.so,
loaded through GCD_LIB_PATH) and the default fp16 library do not overwrite each other.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["gemm.cu", "norm.cu", "elem.cu", "attn_temporal.cu", "attn_spatial.cu", "metrics.cu", "clip.cu", "render.cu", "lpips.cu"]
OUT = os.path.join(HERE, "libgcd_b200.so")


def _stale(out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "gcd_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, bf16=False, verbose=False, out=None):
    out = os.path.abspath(out) if out else OUT
    if not force and not _stale(out):
        return out
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objdir = os.path.join(HERE, "build", "bf16" if bf16 else "fp16")
    objs = []
    procs = []
    os.makedirs(objdir, exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
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
        log, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {src}\n{log}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    subprocess.check_call([nvcc, "-shared", "-Wno-deprecated-gpu-targets", "-o", out] + objs + ["-lcudart_static", "-ldl", "-lrt", "-lpthread"])
    return out


if __name__ == "__main__":
    a = sys.argv[1:]
    print(build(force=True, bf16="--bf16" in a, verbose="--verbose" in a, out=a[a.index("--out") + 1] if "--out" in a else None))
