"""OpenCLIP ViT-H/14 image tower of the GCD conditioner (`FrozenOpenCLIPImageEmbedder`, encoders/modules.py:653-815) on this
package's kernels: open_clip 2.23.0 `VisionTransformer.forward` after kornia 0.7.0 preprocessing.

    patches   = clip_preprocess(x)                 clip.cu: kornia resize (Gaussian antialias + bicubic) -> (x+1)/2 -> normalise
                                                   -> conv1 patch unfold, act [n*257, 640], row 0 of every image zero
    tok       = patches @ conv1^T                  tc_gemm (K = 640), fp32
    x         = ln_pre(tok + pos')                 gcd_layernorm_f32, pos' = positional_embedding with the class embedding
                                                   folded into row 0 (add index row % 257): the fp32 residual stream
    32 x      x += out_proj(attn(ln_1(x)))         gcd_layernorm -> tc_gemm QKV (+bias) -> gcd_attention_d80 -> tc_gemm (+res1)
              x += c_proj(gelu(c_fc(ln_2(x))))     tc_gemm with the exact-GELU epilogue (act 2) -> tc_gemm (+res1)
    z         = ln_post(x[:, 0]) @ proj            class rows gathered, gcd_layernorm, tc_gemm (proj packed transposed)

16-bit tensor-core operands, fp32 accumulation, residual stream and softmax. There is no CPU path.
"""
import torch

from . import ops
from .unet import BufferPool

VIT_H14 = dict(width=1280, layers=32, heads=16, patch=14, image=224, embed=1024)
# Test-size tower with the same head width, patch and image size. Width 320: gcd_layernorm needs C % 64 == 0 and the attention
# kernel 80-wide heads.
VIT_TINY = dict(VIT_H14, width=320, layers=2, heads=4)
# The text side of open_clip's CLIP that `del model.transformer` leaves in the state dict (ViT-H-14: width 1024, 77 tokens).
TEXT_LEFTOVERS_H14 = {"token_embedding.weight": (49408, 1024), "positional_embedding": (77, 1024), "ln_final.weight": (1024,),
                      "ln_final.bias": (1024,), "text_projection": (1024, 1024), "logit_scale": ()}
OPENAI_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_STD = (0.26862954, 0.26130258, 0.27577711)
TOKENS = 257                      # (224 / 14)^2 patches + the class token
PATCH_K = 640                     # 14*14*3 = 588 patch values, zero-padded to a multiple of 64


def visual_param_shapes(cfg):
    """Keys below `model.visual.` and shapes of open_clip's VisionTransformer for `cfg` (ls / attn_pool absent, no conv bias)."""
    w, p, e = cfg["width"], cfg["patch"], cfg["embed"]
    grid = cfg["image"] // p
    d = {"conv1.weight": (w, 3, p, p), "class_embedding": (w,), "positional_embedding": (grid * grid + 1, w),
         "ln_pre.weight": (w,), "ln_pre.bias": (w,)}
    for i in range(cfg["layers"]):
        b = f"transformer.resblocks.{i}."
        d.update({b + "ln_1.weight": (w,), b + "ln_1.bias": (w,),
                  b + "attn.in_proj_weight": (3 * w, w), b + "attn.in_proj_bias": (3 * w,),
                  b + "attn.out_proj.weight": (w, w), b + "attn.out_proj.bias": (w,),
                  b + "ln_2.weight": (w,), b + "ln_2.bias": (w,),
                  b + "mlp.c_fc.weight": (4 * w, w), b + "mlp.c_fc.bias": (4 * w,),
                  b + "mlp.c_proj.weight": (w, 4 * w), b + "mlp.c_proj.bias": (w,)})
    d.update({"ln_post.weight": (w,), "ln_post.bias": (w,), "proj": (w, e)})
    return d


def kornia_blur_taps(H, W, size=224):
    """Antialias taps of kornia 0.7.0 `geometry.resize(..., antialias=True)` for an H x W input resized to size x size:
    (taps along W, taps along H) as float32 CPU tensors, or None when no blur applies (no downscale, or no resize at all).
    sigma_i = max((factor_i - 1) / 2, 0.001), ks_i = int(max(4 sigma_i, 3)) made odd, taps exp(-x^2 / (2 sigma^2)) / sum with
    x = arange(ks) - ks // 2, evaluated in float32 as kornia's `gaussian` does."""
    if (H, W) == (size, size):
        return None
    factors = (H / size, W / size)
    if max(factors) <= 1:
        return None
    sigmas = (max((factors[0] - 1.0) / 2.0, 0.001), max((factors[1] - 1.0) / 2.0, 0.001))
    ks = [int(max(2.0 * 2 * sigmas[0], 3)), int(max(2.0 * 2 * sigmas[1], 3))]
    ks = [k + 1 if k % 2 == 0 else k for k in ks]
    sigma = torch.tensor([list(sigmas)], dtype=torch.float32)

    def gaussian(k, s):
        x = torch.arange(k, dtype=torch.float32) - k // 2
        g = torch.exp(-x.pow(2.0) / (2 * s.pow(2)))
        return (g / g.sum(-1, keepdim=True)).reshape(-1)

    return gaussian(ks[1], sigma[:, 1:2]), gaussian(ks[0], sigma[:, 0:1])


class ClipEngine:
    """Packed weights + workspaces of one tower on one device. `sd`: the VisionTransformer state dict (visual_param_shapes)."""

    def __init__(self, cfg, sd, device):
        self.cfg, self.device = dict(cfg), torch.device(device)
        self.AD = ops.act_dtype()
        w = cfg["width"]
        assert w % 80 == 0 and w % 64 == 0 and cfg["patch"] == 14 and cfg["image"] == 224, "only 224px / patch 14 / 80-wide heads"
        assert w // 80 == cfg["heads"], "head width must be 80"
        f32 = lambda t: t.detach().to(self.device, torch.float32).contiguous()
        act = lambda t: t.detach().to(self.device, torch.float32).to(self.AD).contiguous()
        cw = sd["conv1.weight"].detach().float().permute(0, 2, 3, 1).reshape(w, -1)      # (ky, kx, c) = the patch column order
        self.w_patch = act(torch.nn.functional.pad(cw, (0, PATCH_K - cw.shape[1])))
        pos = sd["positional_embedding"].detach().float().clone()
        pos[0] += sd["class_embedding"].detach().float()
        self.pos = f32(pos)
        self.ln_pre = (f32(sd["ln_pre.weight"]), f32(sd["ln_pre.bias"]))
        self.layers = []
        for i in range(cfg["layers"]):
            b = f"transformer.resblocks.{i}."
            g = lambda k: sd[b + k]
            self.layers.append(dict(
                ln1=(f32(g("ln_1.weight")), f32(g("ln_1.bias"))), ln2=(f32(g("ln_2.weight")), f32(g("ln_2.bias"))),
                w_qkv=act(g("attn.in_proj_weight")), b_qkv=f32(g("attn.in_proj_bias")),
                w_o=act(g("attn.out_proj.weight")), b_o=f32(g("attn.out_proj.bias")),
                w_fc=act(g("mlp.c_fc.weight")), b_fc=f32(g("mlp.c_fc.bias")),
                w_pr=act(g("mlp.c_proj.weight")), b_pr=f32(g("mlp.c_proj.bias"))))
        self.ln_post = (f32(sd["ln_post.weight"]), f32(sd["ln_post.bias"]))
        self.proj_t = act(sd["proj"].detach().float().t())                                # [embed, width]
        self.mean_std = torch.tensor(OPENAI_MEAN + OPENAI_STD, dtype=torch.float32, device=self.device)
        self.pool = BufferPool(self.device)
        self._taps = {}

    def taps(self, H, W):
        if (H, W) not in self._taps:
            t = kornia_blur_taps(H, W)
            self._taps[(H, W)] = None if t is None else tuple(v.to(self.device) for v in t)
        return self._taps[(H, W)]

    def preprocess(self, x):
        """x: float32 [n, 3, H, W] on the device -> act patch matrix [n*257, 640] (a pool buffer)."""
        n, _, H, W = x.shape
        taps = self.taps(H, W)
        out = self.pool.get("patches", (n * TOKENS, PATCH_K), self.AD)
        scratch = self.pool.get("pre_scratch", (2 * x.numel(),), torch.float32) if taps is not None else None
        ops.clip_preprocess(x, taps[0] if taps else None, taps[1] if taps else None, self.mean_std, out, scratch)
        return out

    def forward(self, x):
        """x: float32 [n, 3, H, W] in [-1, 1] on the device -> float32 [n, embed] (pooled, projected)."""
        n = x.shape[0]
        w, heads = self.cfg["width"], self.cfg["heads"]
        rows = n * TOKENS
        P, AD = self.pool, self.AD
        patches = self.preprocess(x.to(torch.float32).contiguous())
        tok = P.get("tok", (rows, w), torch.float32)
        ops.linear(patches, self.w_patch, ops.make_ep(tok))
        res = P.get("res", (rows, w), torch.float32)
        ops.layernorm_f32(tok, *self.ln_pre, res, add=self.pos, add_rows_per=1, add_mod=TOKENS)
        h = P.get("h", (rows, w), AD)
        qkv = P.get("qkv", (rows, 3 * w), AD)
        att = P.get("att", (rows, w), AD)
        mlp = P.get("mlp", (rows, 4 * w), AD)
        for L in self.layers:
            ops.layernorm(res, *L["ln1"], h)
            ops.linear(h, L["w_qkv"], ops.make_ep(qkv, bias=L["b_qkv"]))
            ops.attention_d80(qkv, n, TOKENS, heads, att)
            ops.linear(att, L["w_o"], ops.make_ep(res, bias=L["b_o"], res1=res))
            ops.layernorm(res, *L["ln2"], h)
            ops.linear(h, L["w_fc"], ops.make_ep(mlp, bias=L["b_fc"], act=2))
            ops.linear(mlp, L["w_pr"], ops.make_ep(res, bias=L["b_pr"], res1=res))
        cls = res.view(n, TOKENS, w)[:, 0].contiguous()                        # the n class rows only
        hp = P.get("post", (n, w), AD)
        ops.layernorm(cls, *self.ln_post, hp)
        z = torch.empty(n, self.cfg["embed"], device=self.device, dtype=torch.float32)
        ops.linear(hp, self.proj_t, ops.make_ep(z))
        return z
