"""Per-kernel-class / per-shape CUDA-event breakdown of one CFG UNet forward and one VAE decode at full size."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from gcd_b200 import ops, spec, synthetic
from gcd_b200.pipeline import GCDHotPath

T, H, W = 14, 72, 128
pipe = GCDHotPath(spec.UNET_KUBRIC, spec.VAE_DECODER, num_steps=2, device="cuda")
pipe.load_state(synthetic.seeded_state(spec.unet_param_shapes(spec.UNET_KUBRIC)), synthetic.seeded_state(spec.decoder_param_shapes(spec.VAE_DECODER)))
x, c, uc, _ = synthetic.seeded_inputs(spec.UNET_KUBRIC, 1, T, H, W)
dev = "cuda"
x, c, uc = x.to(dev), {k: v.to(dev) for k, v in c.items()}, {k: v.to(dev) for k, v in uc.items()}
for _ in range(2):
    z = pipe.sample_latents(x.clone(), c, uc)
    fr = pipe.decode_first_stage(z)
ops.DETAIL = True
out = {}
for name, fn in (("unet_2steps", lambda: pipe.sample_latents(x.clone(), c, uc)), ("vae_decode", lambda: pipe.decode_first_stage(z))):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ops.profile() as prof:
        e0.record(); fn(); e1.record()
    summ = prof.summary()
    tot = e0.elapsed_time(e1)
    rows = sorted(summ.items(), key=lambda kv: -kv[1]["ms"])
    print(f"== {name}: wall {tot:.1f} ms, sum of classes {sum(d['ms'] for d in summ.values()):.1f} ms")
    for k, d in rows[:45]:
        print(f"{d['ms']:8.2f} ms  x{d['launches']:4d}  {d['flops']/max(d['ms'],1e-9)/1e9:7.0f} TF  {d['bytes']/max(d['ms'],1e-9)/1e6:7.0f} GB/s  {k}")
    out[name] = {"wall_ms": tot, "classes": {k: d for k, d in rows}}
# Practical ceiling of this card at its power limit: cuBLAS fp16 at three of the UNet's linear shapes (a yardstick for the table
# above only; nothing in the package calls cuBLAS).
out["cublas_ceiling"] = {}
for M, K, N in ((258048, 320, 2560), (258048, 1280, 320), (64512, 640, 5120)):
    a = torch.randn(M, K, device=dev, dtype=torch.float16)
    b = torch.randn(N, K, device=dev, dtype=torch.float16)
    for _ in range(5):
        torch.matmul(a, b.t())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        torch.matmul(a, b.t())
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    print(f"cuBLAS fp16 M{M} N{N} K{K}: {ms:.3f} ms  {2.0 * M * N * K / ms / 1e9:.0f} TF")
    out["cublas_ceiling"][f"M{M} N{N} K{K}"] = {"ms": ms, "tflops": 2.0 * M * N * K / ms / 1e9}
    del a, b
import subprocess
print("card:", torch.cuda.get_device_name(0), "power limit:", subprocess.run(
    ["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
os.makedirs("gpurun_out", exist_ok=True)
json.dump(out, open("gpurun_out/prof_forward.json", "w"), indent=1)
