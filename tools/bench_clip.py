"""OpenCLIP ViT-H/14 image tower of the conditioner on 14 frames (at 256x384 and 576x1024): CUDA-event time per call after a
warm-up, TFLOP/s from the shapes, and the card's name and power limit.

    python tools/bench_clip.py [--iters N]
"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from gcd_b200 import clip, synthetic  # noqa: E402
from gcd_b200.embedders import FrozenOpenCLIPImageEmbedder  # noqa: E402


def tower_flop(n, cfg=clip.VIT_H14):
    """2 * MAC of the tower for n frames: patch embedding, per layer QKV / attention / out_proj / MLP, final proj."""
    w, L, T = cfg["width"], cfg["layers"], clip.TOKENS
    per_layer = 2 * T * w * 3 * w + 2 * 2 * T * T * w + 2 * T * w * w + 2 * 2 * T * w * 4 * w
    return n * (2 * T * 588 * w + L * per_layer + 2 * w * cfg["embed"])


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def main():
    iters = int(sys.argv[sys.argv.index("--iters") + 1]) if "--iters" in sys.argv else 10
    emb = FrozenOpenCLIPImageEmbedder()
    sd = synthetic.seeded_state(clip.visual_param_shapes(clip.VIT_H14), seed=0)
    emb.load_state_dict({"model.visual." + k: v for k, v in sd.items()}, strict=False)
    emb = emb.cuda()
    name, pl = card()
    print(f"card: {name}, power limit {pl}")
    for n, H, W in [(14, 256, 384), (14, 576, 1024)]:
        x = torch.rand(n, 3, H, W, device="cuda") * 2 - 1
        for _ in range(3):
            z = emb(x)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            z = emb(x)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        fl = tower_flop(n)
        print(f"ViT-H/14 {n}x3x{H}x{W} -> {tuple(z.shape)}: {ms:.2f} ms, {fl / 1e12:.2f} TFLOP, {fl / ms / 1e9:.0f} TFLOP/s "
              f"(finite={bool(torch.isfinite(z).all())})")


if __name__ == "__main__":
    main()
