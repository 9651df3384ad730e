"""fp32 torch restatement of the LPIPS perceptual distance, VGG16 variant (gcd-model/sgm/modules/autoencoding/lpips/loss/lpips.py):
ScalingLayer, torchvision's vgg16().features[:30] cut after relu1_2 / relu2_2 / relu3_3 / relu4_3 / relu5_3, unit-normalised feature
differences and the `lin` 1x1 heads, spatially averaged. Written with F.conv2d / F.relu / F.max_pool2d only (no torchvision), so it
runs wherever the tests do, on CPU or on the GPU; TF32 is switched off for the convolutions.

Also the seeded weights and inputs of the goldens (oracle/pin_lpips.py) and of the GPU tests."""
import math

import torch
import torch.nn.functional as F

CHNS = (64, 128, 256, 512, 512)
SLICES = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))
SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)


def seeded_state(seed=0):
    """A reference-keyed LPIPS state dict: He-normal convs (std sqrt(2 / fan_in)), small biases, non-negative `lin` weights (LPIPS
    clamps its trained linear weights to >= 0), the real ScalingLayer constants."""
    g = torch.Generator().manual_seed(seed)
    sd, cin = {}, 3
    for k, (idx, cout) in enumerate(zip(SLICES, CHNS)):
        for i in idx:
            sd[f"net.slice{k + 1}.{i}.weight"] = torch.randn(cout, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
            sd[f"net.slice{k + 1}.{i}.bias"] = torch.randn(cout, generator=g) * 0.05
            cin = cout
    for k, c in enumerate(CHNS):
        sd[f"lin{k}.model.1.weight"] = torch.rand(1, c, 1, 1, generator=g)
    sd["scaling_layer.shift"] = torch.tensor(SHIFT)[None, :, None, None]
    sd["scaling_layer.scale"] = torch.tensor(SCALE)[None, :, None, None]
    return sd


def features(sd, x):
    """The five tapped VGG16 activations of x [n, 3, H, W] in [-1, 1]."""
    h = (x - sd["scaling_layer.shift"].to(x)) / sd["scaling_layer.scale"].to(x)
    outs = []
    with torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
        for k, idx in enumerate(SLICES):
            if k > 0:
                h = F.max_pool2d(h, 2, 2)
            for i in idx:
                h = F.relu(F.conv2d(h, sd[f"net.slice{k + 1}.{i}.weight"].to(x), sd[f"net.slice{k + 1}.{i}.bias"].to(x), padding=1))
            outs.append(h)
    return outs


def layer_terms(sd, x, y):
    """Per-layer LPIPS terms, float32 [5, n]: spatial mean of lin_k((x_k / |x_k| - y_k / |y_k|)^2)."""
    terms = []
    for k, (a, b) in enumerate(zip(features(sd, x), features(sd, y))):
        a = a / (torch.sqrt(torch.sum(a ** 2, dim=1, keepdim=True)) + 1e-10)
        b = b / (torch.sqrt(torch.sum(b ** 2, dim=1, keepdim=True)) + 1e-10)
        d = F.conv2d((a - b) ** 2, sd[f"lin{k}.model.1.weight"].to(x))
        terms.append(d.mean([2, 3])[:, 0])
    return torch.stack(terms)


def lpips(sd, x, y):
    """LPIPS(x, y), float32 [n] (the reference's [n, 1, 1, 1] flattened)."""
    t = layer_terms(sd, x, y)
    v = t[0]
    for k in range(1, 5):
        v = v + t[k]
    return v


def smooth_field(n, H, W, g, cells=(6, 8)):
    """n smooth images in [-1, 1]: seeded coarse noise, bicubic-upsampled, plus a little fine noise."""
    c = torch.randn(n, 3, cells[0], cells[1], generator=g)
    x = F.interpolate(c, size=(H, W), mode="bicubic", align_corners=False)
    x = x + 0.05 * torch.randn(n, 3, H, W, generator=g)
    return torch.tanh(0.8 * x)


def pair_inputs(n, H, W, seed):
    """(pred, gt) in [-1, 1]: gt a smooth field; pred a perturbed gt, shifted by a few pixels in its right half."""
    g = torch.Generator().manual_seed(seed)
    gt = smooth_field(n, H, W, g)
    pred = gt.clone()
    s = 1 + int(torch.randint(0, 4, (1,), generator=g))
    pred[..., W // 2:] = torch.roll(gt, shifts=(s, s), dims=(2, 3))[..., W // 2:]
    pred = pred + 0.3 * smooth_field(n, H, W, g, (4, 5)) + 0.05 * torch.randn(n, 3, H, W, generator=g)
    return pred.clamp(-1, 1), gt
