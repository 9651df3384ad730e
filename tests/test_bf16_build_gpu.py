"""The bf16 build of the library (-DGCD_ACT_BF16: bf16 tensor-core operands, bf16 activations and 16-bit outputs).

The module fixture builds it next to the default library as gcd_b200/libgcd_b200_bf16.so (objects under gcd_b200/build/bf16/;
an up-to-date library is reused) and the tests run child Pythons that load it through GCD_LIB_PATH: one GEMM and the dtype
guards directly, then the kernel parity suites (test_ops_gpu.py, test_tc_pingpong_gpu.py, test_tc_accumulation_gpu.py,
test_attention_edges_gpu.py, test_lpips_gpu.py and the op tests of test_clip_gpu.py), whose per-element bounds follow the operand type
(oracle/error_model.py).

The model-level goldens (UNet, VAE, CLIP tower, sampler trajectories) are not run on the bf16 build: their bars are fitted to
fp16 as the reference runs it, and bf16 tolerances for whole models are not stated.
"""
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16_LIB = os.path.join(ROOT, "gcd_b200", "libgcd_b200_bf16.so")
CLIP_OP_TESTS = ["test_preprocess_vs_golden", "test_attention_d80_vs_sdpa", "test_gelu_epilogue",
                 "test_layernorm_f32_with_position_add"]


@pytest.fixture(scope="module")
def bf16_env():
    from gcd_b200 import build
    path = build.build(bf16=True, out=BF16_LIB)
    env = dict(os.environ, GCD_LIB_PATH=path, PYTHONDONTWRITEBYTECODE="1")
    return env


def _python():
    return [sys.executable] + (["-s"] if sys.flags.no_user_site else [])


CHILD = r"""
import torch
from gcd_b200 import _lib, ops
from oracle import error_model as EM
ops.lib()
assert not _lib.MISSING, _lib.MISSING
assert ops.act_dtype() == torch.bfloat16, ops.act_dtype()
g = torch.Generator().manual_seed(7)
M, K, N = 300, 320, 320
x = torch.randn(M, K, generator=g).to(torch.bfloat16).cuda()
w = (torch.randn(N, K, generator=g) * K ** -0.5).to(torch.bfloat16).cuda()
b = torch.randn(N, generator=g).cuda()
try:
    ops.make_ep(torch.empty(M, N, device="cuda", dtype=torch.float16))
    raise SystemExit("an fp16 output was accepted by the bf16 build")
except _lib.GcdError:
    pass
try:
    ops.linear(x.half(), w.half(), ops.make_ep(torch.empty(M, N, device="cuda")))
    raise SystemExit("fp16 operands were accepted by the bf16 build")
except AssertionError:
    pass
out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
ops.linear(x, w, ops.make_ep(out, bias=b))
EM.check(out, x.double() @ w.double().t() + b.double(), EM.gemm_scale(x, w, b), "gemm", "bf16 build linear")
print("child ok")
"""


def test_bf16_library_loads_and_computes(bf16_env):
    r = subprocess.run(_python() + ["-c", CHILD], cwd=ROOT, env=bf16_env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "child ok" in r.stdout, r.stdout + r.stderr


def test_bf16_kernel_parity_suite(bf16_env):
    targets = ["tests/test_ops_gpu.py", "tests/test_tc_pingpong_gpu.py", "tests/test_tc_accumulation_gpu.py",
               "tests/test_attention_edges_gpu.py", "tests/test_lpips_gpu.py"]
    targets += [f"tests/test_clip_gpu.py::{t}" for t in CLIP_OP_TESTS]
    r = subprocess.run(_python() + ["-m", "pytest", "-q", "-s", "-p", "no:cacheprovider"] + targets, cwd=ROOT, env=bf16_env,
                       capture_output=True, text=True, timeout=3000)
    ratios = "\n".join(line[line.index("error/bound"):] for line in r.stdout.splitlines() if "error/bound" in line)
    print(ratios)
    tail = r.stdout[-3000:] + r.stderr[-3000:]
    assert r.returncode == 0, tail
    summary = r.stdout.strip().splitlines()[-1]
    assert re.search(r"\d+ passed", summary) and "skipped" not in summary and "deselected" not in summary, summary
