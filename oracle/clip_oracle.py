"""fp32 PyTorch restatement of the conditioner's image tower (TEST INFRASTRUCTURE, CPU only): kornia 0.7.0 preprocessing and
open_clip 2.23.0 `VisionTransformer.forward` for the ViT-H/14 layout (gcd_b200/clip.py). Neither package is installed
anywhere this project is tested, so their arithmetic is restated here from their documented behaviour; the reference's own
wrapper code (FrozenOpenCLIPImageEmbedder, FrozenOpenCLIPImagePredictionEmbedder, GeneralConditioner) runs on top of these
pieces in oracle/pin_clip.py."""
import torch
import torch.nn.functional as F


def kornia_gaussian(k, sigma):
    """kornia.filters.kernels.gaussian (0.7.0) for one float32 sigma."""
    s = torch.tensor([[sigma]], dtype=torch.float32)
    x = torch.arange(k, dtype=torch.float32) - k // 2
    if k % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * s.pow(2)))
    return (g / g.sum(-1, keepdim=True)).reshape(-1)


def kornia_resize(x, size=(224, 224), interpolation="bicubic", align_corners=True, antialias=True):
    """kornia.geometry.resize (0.7.0) for NCHW float32 input: optional Gaussian antialias blur (separable, horizontal first,
    'reflect' border), then torch bicubic interpolation."""
    size = tuple(size)
    h, w = x.shape[-2:]
    if size == (h, w):
        return x
    factors = (h / size[0], w / size[1])
    if antialias and max(factors) > 1:
        sigmas = (max((factors[0] - 1.0) / 2.0, 0.001), max((factors[1] - 1.0) / 2.0, 0.001))
        ks = [int(max(2.0 * 2 * sigmas[0], 3)), int(max(2.0 * 2 * sigmas[1], 3))]
        ks = [k + 1 if k % 2 == 0 else k for k in ks]
        kx, ky = kornia_gaussian(ks[1], sigmas[1]), kornia_gaussian(ks[0], sigmas[0])
        c = x.shape[1]
        x = F.conv2d(F.pad(x, (ks[1] // 2, ks[1] // 2, 0, 0), mode="reflect"), kx.view(1, 1, 1, -1).expand(c, 1, 1, -1),
                     groups=c)
        x = F.conv2d(F.pad(x, (0, 0, ks[0] // 2, ks[0] // 2), mode="reflect"), ky.view(1, 1, -1, 1).expand(c, 1, -1, 1),
                     groups=c)
    return F.interpolate(x, size=size, mode=interpolation, align_corners=align_corners)


def kornia_normalize(x, mean, std):
    """kornia.enhance.normalize (0.7.0)."""
    mean = torch.as_tensor(mean, dtype=x.dtype).view(1, -1, 1, 1)
    std = torch.as_tensor(std, dtype=x.dtype).view(1, -1, 1, 1)
    return (x - mean) / std


OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)


def clip_preprocess(x):
    """FrozenOpenCLIPImageEmbedder.preprocess (encoders/modules.py:703-715): [n, 3, H, W] in [-1, 1] -> [n, 3, 224, 224]."""
    x = kornia_resize(x, (224, 224), interpolation="bicubic", align_corners=True, antialias=True)
    x = (x + 1.0) / 2.0
    return kornia_normalize(x, torch.tensor(OPENAI_MEAN), torch.tensor(OPENAI_STD))


def clip_visual_forward(sd, cfg, img):
    """open_clip 2.23.0 VisionTransformer.forward (no attention pool, 'tok' pooling): sd holds the `visual.` keys of
    gcd_b200.clip.visual_param_shapes; img is the preprocessed [n, 3, 224, 224] batch -> [n, embed]."""
    w, heads, p = cfg["width"], cfg["heads"], cfg["patch"]
    x = F.conv2d(img, sd["conv1.weight"], stride=p)                                   # conv1, no bias
    x = x.reshape(x.shape[0], x.shape[1], -1).permute(0, 2, 1)
    cls = sd["class_embedding"].view(1, 1, w).expand(x.shape[0], -1, -1)
    x = torch.cat([cls, x], dim=1) + sd["positional_embedding"]
    x = F.layer_norm(x, (w,), sd["ln_pre.weight"], sd["ln_pre.bias"])
    x = x.permute(1, 0, 2)                                                            # NLD -> LND (nn.MultiheadAttention)
    for i in range(cfg["layers"]):
        b = f"transformer.resblocks.{i}."
        g = lambda k: sd[b + k]
        h = F.layer_norm(x, (w,), g("ln_1.weight"), g("ln_1.bias"))
        a, _ = F.multi_head_attention_forward(h, h, h, w, heads, g("attn.in_proj_weight"), g("attn.in_proj_bias"), None, None,
                                              False, 0.0, g("attn.out_proj.weight"), g("attn.out_proj.bias"),
                                              training=False, need_weights=False)
        x = x + a
        h = F.layer_norm(x, (w,), g("ln_2.weight"), g("ln_2.bias"))
        x = x + F.linear(F.gelu(F.linear(h, g("mlp.c_fc.weight"), g("mlp.c_fc.bias"))), g("mlp.c_proj.weight"),
                         g("mlp.c_proj.bias"))
    x = x.permute(1, 0, 2)
    pooled = F.layer_norm(x[:, 0], (w,), sd["ln_post.weight"], sd["ln_post.bias"])
    return pooled @ sd["proj"]


def clip_image_embed(sd, cfg, frames):
    """The whole tower: frames [n, 3, H, W] in [-1, 1] -> [n, embed]."""
    return clip_visual_forward(sd, cfg, clip_preprocess(frames))
