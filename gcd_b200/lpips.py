"""LPIPS perceptual distance, VGG16 variant (gcd-model/sgm/modules/autoencoding/lpips/loss/lpips.py), on the device: the metric
that DiffusionEngine.validation_step logs next to PSNR and SSIM (models/diffusion.py:317-362).

`LPIPS` has the reference module's parameter and buffer names and shapes (`net.slice<k>.<i>.weight/bias`, `lin<k>.model.1.weight`,
`scaling_layer.shift/scale`), so the `lpips.*` tensors of a DiffusionEngine state dict load into it (checkpoint.HotPathRoot). The
constructor downloads nothing and does not import torchvision: the weights arrive through `load_state_dict`.

Per chunk of frames (csrc/lpips.cu, tc_gemm): the input stage (ScalingLayer + conv1_1's im2col) -> 13 tensor-core convs with a fused
bias + ReLU epilogue, a 2x2 max-pool before the convs of slices 2..5 -> after each slice one fused head launch that adds the
layer's term of every (input, target) pair to a float64 result. No CPU or eager-PyTorch path."""
import torch
import torch.nn as nn

from . import ops
from .engine import Engine, EngineCache, _Node, register_param_tree

CHNS = (64, 128, 256, 512, 512)
# torchvision vgg16().features indices of the convolutions, per slice (slice1 = features[0:4], ..., slice5 = features[23:30])
SLICES = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
ROWS_PER_CHUNK = 1 << 22      # pixels (frames x H x W) per chunk: two 16-bit buffers of 64 channels, 0.5 GiB each


def param_shapes():
    """Parameter names and shapes of the reference LPIPS (buffers excluded)."""
    shapes, cin = {}, 3
    for k, (idx, cout) in enumerate(zip(SLICES, CHNS)):
        for i in idx:
            shapes[f"net.slice{k + 1}.{i}.weight"] = (cout, cin, 3, 3)
            shapes[f"net.slice{k + 1}.{i}.bias"] = (cout,)
            cin = cout
    for k, c in enumerate(CHNS):
        shapes[f"lin{k}.model.1.weight"] = (1, c, 1, 1)
    return shapes


class LPIPSEngine(Engine):
    """Packed VGG16 convolutions (16-bit [Cout, (ky, kx, c)], fp32 biases) and `lin` weights of one LPIPS module on one device."""

    def __init__(self, sd, device):
        super().__init__(device)
        for k, idx in enumerate(SLICES):
            for i in idx:
                key = f"net.slice{k + 1}.{i}"
                if i == 0:      # conv1_1 over the input stage's im2col: [64, 3, 3, 3] -> [64, (ky, kx, c)], 27 columns padded to 64
                    self._put(sd, key, key, lambda w: torch.cat([w.permute(0, 2, 3, 1).reshape(w.shape[0], 27),
                                                                 w.new_zeros(w.shape[0], 37)], 1))
                else:
                    self._conv3(sd, key, key)
            self.w[f"lin{k}"] = self._f32(sd[f"lin{k}.model.1.weight"]).reshape(-1).contiguous()
        self.count = torch.zeros(0, device=self.device, dtype=torch.int32)

    def _conv(self, key, x, out):
        ops.conv2d_3x3(x, self.w[key + ".w"], ops.make_ep(out.view(-1, out.shape[-1]), bias=self.w[key + ".b"], act=3))

    def distances(self, frames, pairs, shift, scale):
        """frames: float32 [F, 3, H, W] in [-1, 1] on the device; pairs: int32 [P, 2] frame indices on the device.
        Returns float64 [5, P]: the term of each tapped layer (relu1_2 .. relu5_3) for each pair."""
        F_, _, H, W = frames.shape
        P = pairs.shape[0]
        numel = F_ * H * W * 64                   # the largest activation of the pass (relu1_*; deeper layers are smaller)
        bufs = [self.pool.get(n, (numel,), self.AD) for n in ("lp_a", "lp_b")]
        partial = self.pool.get("lp_partial", (P * ((H * W + ops.LPIPS_HEAD_PIX - 1) // ops.LPIPS_HEAD_PIX),), torch.float64)
        if self.count.numel() < P:                            # the head's per-pair counters are zeroed once; each launch leaves them zero
            self.count = torch.zeros(P, device=self.device, dtype=torch.int32)
        out = torch.empty(5, P, device=self.device, dtype=torch.float64)

        def view(i, h, w, c):
            return bufs[i][:F_ * h * w * c].view(F_, h, w, c)

        ops.lpips_input(frames, shift, scale, bufs[0][:F_ * H * W * 64].view(-1, 64))
        cur, h, w, cin = 0, H, W, 64
        for k, idx in enumerate(SLICES):
            if k > 0:
                ops.maxpool2x2(view(cur, h, w, cin), view(1 - cur, h // 2, w // 2, cin))
                cur, h, w = 1 - cur, h // 2, w // 2
            for i in idx:
                key = f"net.slice{k + 1}.{i}"
                cout = self.w[key + ".w"].shape[0]
                if i == 0:
                    ops.linear(bufs[cur][:F_ * h * w * 64].view(-1, 64), self.w[key + ".w"],
                               ops.make_ep(bufs[1 - cur][:F_ * h * w * cout].view(-1, cout), bias=self.w[key + ".b"], act=3))
                else:
                    self._conv(key, view(cur, h, w, cin), view(1 - cur, h, w, cout))
                cur, cin = 1 - cur, cout
            ops.lpips_head(bufs[cur][:F_ * h * w * cin].view(F_, h * w, cin), pairs, self.w[f"lin{k}"], partial, self.count, out[k])
        return out


class LPIPS(nn.Module):
    """Drop-in for the reference `LPIPS` (eval mode). forward(input, target): CUDA float32 [n, 3, H, W] in [-1, 1] ->
    float32 [n, 1, 1, 1]. H and W must be at least 16 (four 2x2 pools before relu5_3)."""

    def __init__(self):
        super().__init__()
        register_param_tree(self, param_shapes())
        for p in self.parameters():
            p.requires_grad_(False)
        self.scaling_layer = _Node()
        self.scaling_layer.register_buffer("shift", torch.tensor(SHIFT)[None, :, None, None])
        self.scaling_layer.register_buffer("scale", torch.tensor(SCALE)[None, :, None, None])
        self._engines = EngineCache()

    def engine(self, device):
        return self._engines.get(self, device, lambda: LPIPSEngine(self.state_dict(), device))

    def layer_distances(self, input, target):
        """Per-layer LPIPS terms, float64 [5, N] on the device. input: [N, 3, H, W]; target: [M, 3, H, W] with N == M (pair i is
        (input[i], target[i])) or N == S * M (pair i is (input[i], target[i % M]): the target's features are computed once, not S
        times). Frames are processed in chunks of whole target frames with their S inputs."""
        for name, t in (("input", input), ("target", target)):
            if t.dim() != 4 or t.shape[1] != 3 or not t.is_floating_point():
                raise ValueError(f"LPIPS: {name} must be a float [n, 3, H, W] tensor, got {tuple(t.shape)} {t.dtype}")
        N, M = input.shape[0], target.shape[0]
        if input.shape[2:] != target.shape[2:] or M == 0 or N % M != 0:
            raise ValueError(f"LPIPS: input {tuple(input.shape)} and target {tuple(target.shape)} do not pair up")
        H, W = input.shape[2:]
        if H < 16 or W < 16:
            raise ValueError(f"LPIPS: frames of {H}x{W} are too small for relu5_3 (need at least 16x16)")
        ops._need_cuda(input, target)
        if input.device != target.device:
            raise ValueError("LPIPS: input and target are on different devices")
        S, dev = N // M, input.device
        eng = self.engine(dev)
        shift = self.scaling_layer.shift.to(dev, torch.float32).contiguous()
        scale = self.scaling_layer.scale.to(dev, torch.float32).contiguous()
        x = input.to(torch.float32).reshape(S, M, 3, H, W)
        y = target.to(torch.float32)
        out = torch.empty(5, S, M, device=dev, dtype=torch.float64)
        tc = max(1, ROWS_PER_CHUNK // (H * W) // (S + 1))
        for t0 in range(0, M, tc):
            t1 = min(M, t0 + tc)
            n = t1 - t0
            frames = torch.cat([y[t0:t1], x[:, t0:t1].reshape(S * n, 3, H, W)]).contiguous()
            k = torch.arange(S * n, dtype=torch.int32)
            pairs = torch.stack([n + k, k % n], 1).to(dev)
            out[:, :, t0:t1] = eng.distances(frames, pairs, shift, scale).view(5, S, n)
        return out.view(5, N)

    def forward(self, input, target):
        if input.shape != target.shape:
            raise ValueError(f"LPIPS: input {tuple(input.shape)} and target {tuple(target.shape)} differ in shape")
        return self.layer_distances(input, target).sum(0).to(torch.float32).view(-1, 1, 1, 1)

