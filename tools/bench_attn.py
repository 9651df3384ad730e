"""Times the attention kernels (CUDA events, L2 flushed by the 1.3 GB working set rotation): spatial at the three UNet levels,
temporal (T = 14, 2 clips) at the same levels and the CLIP tower's d80 (14 images x 257 tokens x 16 heads).
GCD_FA_EMU=0|4|2 selects the share of exponentials evaluated on the FMA pipe (read once per process)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gcd_b200 import ops
AD = ops.act_dtype()
torch.manual_seed(0)


def timed(run, n=12):
    for i in range(3):
        run(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        run(i % 3)
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


res = {}
for (f, tok, h) in ((28, 9216, 5), (28, 2304, 10), (28, 576, 20)):
    qkvs = [(torch.randn(f, tok, 3 * h * 64, device="cuda") * 1.0).to(AD) for _ in range(3)]
    out = torch.empty(f, tok, h * 64, device="cuda", dtype=AD)
    ms = timed(lambda i: ops.attention_spatial(qkvs[i], f, tok, h, out))
    fl = 4.0 * f * h * tok * tok * 64
    res[f"spatial {f}x{tok}x{h}"] = (round(ms, 4), round(fl / ms / 1e9, 1))
    # correctness vs torch SDPA (fp32)
    q, k, v = qkvs[0].float().view(f, tok, 3, h, 64).permute(2, 0, 3, 1, 4)[:, :2].unbind(0)
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(2, tok, h * 64)
    ops.attention_spatial(qkvs[0], f, tok, h, out)
    err = ((out[:2].float() - ref).norm() / ref.norm()).item()
    res[f"spatial {f}x{tok}x{h}"] += (f"{err:.2e}",)
    # temporal: the same tensors as 2 clips of T = 14 frames; HBM-bound, so GB/s of qkv read + out written
    ms = timed(lambda i: ops.attention_temporal(qkvs[i], f // 14, 14, tok, h, out))
    res[f"temporal {f}x{tok}x{h} T=14"] = (round(ms, 4), round(f * tok * h * 64 * 2 * 4 / ms / 1e6, 1))
    del qkvs, out
n, L, h = 14, 257, 16
qkvs = [torch.randn(n * L, 3 * h * 80, device="cuda").to(AD) for _ in range(3)]
out = torch.empty(n * L, h * 80, device="cuda", dtype=AD)
ms = timed(lambda i: ops.attention_d80(qkvs[i], n, L, h, out), n=50)
res[f"d80 {n}x{L}x{h}"] = (round(ms, 4), round(4.0 * n * h * L * L * 80 / ms / 1e9, 1))
print("GCD_FA_EMU", os.environ.get("GCD_FA_EMU", "default"), "(ms, TFLOP/s spatial + d80 | GB/s temporal)", res)
