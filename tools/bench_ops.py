"""Micro-benchmarks of the hot kernels at the BASELINE shapes (config 5): run on an H100."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gcd_b200 import ops

AD = ops.act_dtype()
dev = "cuda"
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


res = []


def rep(name, ms, flops=None, bytes_=None):
    d = {"name": name, "ms": round(ms, 4)}
    if flops: d["tflops"] = round(flops / ms / 1e9, 1)
    if bytes_: d["gbs"] = round(bytes_ / ms / 1e6, 1)
    res.append(d); print(json.dumps(d), flush=True)


def rand(*s, dt=AD):
    return (torch.randn(*s, device=dev) * 0.5).to(dt)


sel = sys.argv[1:] or ["linear", "conv", "convt", "attn", "norm"]
if "linear" in sel:
    for (M, K, N, geglu, resid) in [(258048, 320, 320, 0, 1), (258048, 320, 960, 0, 0), (258048, 320, 2560, 1, 0),
                                    (258048, 1280, 320, 0, 1), (64512, 640, 640, 0, 1), (64512, 640, 5120, 1, 0),
                                    (64512, 2560, 640, 0, 1), (16128, 1280, 1280, 0, 1), (16128, 1280, 10240, 1, 0),
                                    (16128, 5120, 1280, 0, 1), (8192, 8192, 8192, 0, 0)]:
        x, w = rand(M, K), rand(N, K)
        No = N // 2 if geglu else N
        out = torch.empty(M, No, device=dev, dtype=torch.float32 if resid else AD)
        ep = ops.make_ep(out, bias=torch.zeros(N, device=dev), res1=out if resid else None, geglu=bool(geglu))
        ms = timeit(lambda: ops.linear(x, w, ep))
        byt = M * K * 2 + N * K * 2 + M * No * (8 if resid else 2)
        rep(f"linear M{M} K{K} N{N} geglu{geglu} res{resid}", ms, 2.0 * M * K * N, byt)
if "conv" in sel:
    for (n, H, W, C, Co) in [(28, 72, 128, 320, 320), (28, 36, 64, 640, 640), (28, 18, 32, 1280, 1280),
                             (28, 9, 16, 1280, 1280), (28, 9, 16, 2560, 1280), (28, 72, 128, 960, 320),
                             (14, 72, 128, 512, 512), (14, 144, 256, 512, 512), (14, 288, 512, 256, 256),
                             (14, 576, 1024, 128, 128)]:
        x, w = rand(n, H, W, C), rand(Co, 9 * C)
        out = torch.empty(n * H * W, Co, device=dev, dtype=AD)
        ep = ops.make_ep(out, bias=torch.zeros(Co, device=dev))
        ms = timeit(lambda: ops.conv2d_3x3(x, w, ep), iters=3)
        rep(f"conv3x3 n{n} {H}x{W} {C}->{Co}", ms, 2.0 * n * H * W * C * Co * 9, n * H * W * (C + Co) * 2)
        del x, w, out
if "convt" in sel:
    for (B, T, HW, C) in [(2, 14, 9216, 320), (2, 14, 2304, 640), (2, 14, 576, 1280), (2, 14, 144, 1280)]:
        x, w = rand(B, T, HW, C), rand(C, 3 * C)
        out = torch.empty(B * T * HW, C, device=dev, dtype=torch.float32)
        ep = ops.make_ep(out, bias=torch.zeros(C, device=dev), res1=out)
        ms = timeit(lambda: ops.conv_t3(x, w, ep))
        rep(f"conv_t3 B{B} T{T} HW{HW} C{C}", ms, 2.0 * B * T * HW * C * C * 3, B * T * HW * C * (2 + 8))
if "attn" in sel:
    for (f, tok, h) in [(28, 9216, 5), (28, 2304, 10), (28, 576, 20), (28, 144, 20)]:
        qkv = rand(f, tok, 3 * h * 64)
        out = torch.empty(f, tok, h * 64, device=dev, dtype=AD)
        ms = timeit(lambda: ops.attention_spatial(qkv, f, tok, h, out), iters=3)
        rep(f"attn_spatial f{f} tok{tok} h{h}", ms, 4.0 * f * h * tok * tok * 64, f * tok * h * 64 * 2 * 4)
    for (clips, tok, h) in [(2, 9216, 5), (2, 2304, 10), (2, 576, 20)]:
        qkv = rand(clips * 14, tok, 3 * h * 64)
        out = torch.empty(clips * 14, tok, h * 64, device=dev, dtype=AD)
        ms = timeit(lambda: ops.attention_temporal(qkv, clips, 14, tok, h, out))
        rep(f"attn_temporal clips{clips} tok{tok} h{h}", ms, 4.0 * clips * tok * h * 14 * 14 * 64, clips * 14 * tok * h * 64 * 2 * 4)
if "norm" in sel:
    for (n, rows, C) in [(28, 9216, 320), (2, 14 * 9216, 320), (28, 2304, 640), (28, 576, 1280)]:
        x = torch.randn(n * rows, C, device=dev)
        g, b = torch.ones(C, device=dev), torch.zeros(C, device=dev)
        out = torch.empty(n * rows, C, device=dev, dtype=AD)
        st = torch.empty(n * 64, device=dev, dtype=torch.float64)
        ms = timeit(lambda: ops.groupnorm(x, n, rows, C, g, b, 1e-5, True, out, st))
        rep(f"groupnorm(stats+apply) n{n} rows{rows} C{C}", ms, None, n * rows * C * (4 + 4 + 2))
        ms = timeit(lambda: ops.layernorm(x, g, b, out))
        rep(f"layernorm rows{n*rows} C{C}", ms, None, n * rows * C * (4 + 2))
os.makedirs("gpurun_out", exist_ok=True)
json.dump(res, open("gpurun_out/bench_ops.json", "w"), indent=1)
