"""Writes the image-tower and conditioning goldens under tests/golden/ (needs a reference checkout: GCD_REFERENCE, see
oracle/ref_shim.py).

    python -m oracle.pin_clip [--full]

The reference's FrozenOpenCLIPImageEmbedder, FrozenOpenCLIPImagePredictionEmbedder, VideoPredictionEmbedderWithEncoder,
ConcatTimestepEmbedderND, SphericalEmbedder and GeneralConditioner are cut out of encoders/modules.py with `ast` and executed,
so their wrapper logic (preprocess order, mean / std, rearrange / repeat, uc zeroing, vector order) is the reference's own.
open_clip and kornia are not installed, so `open_clip.create_model_and_transforms` and `kornia.geometry.resize` /
`kornia.enhance.normalize` are stubs that run the fp32 restatement in oracle/clip_oracle.py: the arithmetic inside those two
packages is the one place where these goldens are not the reference's end to end. The conditioning-frame encoder is the
reference Encoder + quant_conv + DiagonalGaussianDistribution.mode().

Weights and inputs are regenerated from seeds (gcd_b200.synthetic); only outputs are stored. `--full` adds the ViT-H/14
tower (632 M parameters; a few minutes on CPU).
"""
import ast
import math
import os
import sys
import types
import typing
from contextlib import nullcontext

import numpy as np
import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcd_b200 import clip, spec  # noqa: E402
from gcd_b200.sampling import instantiate_from_config  # noqa: E402
from oracle import clip_oracle as CO  # noqa: E402
from oracle import ref_shim, weights  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
torch.set_grad_enabled(False)
SIZES_TINY = [(2, 224, 224), (2, 256, 384), (2, 576, 1024)]
SIZES_FULL = [(14, 256, 384), (2, 576, 1024)]
COND_HW = (64, 96)
COND_FRAMES = 2
PRE_STRIDE = 7                       # preprocessed 224x224 tensors are stored as [..., ::7, ::7]


def frames(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, H, W, generator=g) * 2 - 1


def frame_seed(n, H, W):
    return 1000 + n * 7 + H * 3 + W


def visual_state(cfg, seed=0):
    return weights.seeded_state(clip.visual_param_shapes(cfg), seed=seed)


class _Visual(nn.Module):
    def __init__(self, sd, cfg):
        super().__init__()
        self.sd, self.cfg, self.output_tokens = sd, cfg, False

    def forward(self, img):
        return CO.clip_visual_forward(self.sd, self.cfg, img)


class _StubCLIP(nn.Module):
    def __init__(self, sd, cfg):
        super().__init__()
        self.visual = _Visual(sd, cfg)
        self.transformer = nn.Identity()       # the reference deletes it


def stub_packages(sd, cfg):
    oc = types.ModuleType("open_clip")
    oc.create_model_and_transforms = lambda arch, device=None, pretrained=None: (_StubCLIP(sd, cfg), None, None)
    ko = types.ModuleType("kornia")
    ko.geometry = types.SimpleNamespace(resize=CO.kornia_resize)
    ko.enhance = types.SimpleNamespace(normalize=CO.kornia_normalize)
    return oc, ko


class _RefAEModeOnly(nn.Module):
    """Stands in for sgm.models.autoencoder.AutoencoderKLModeOnly (a LightningModule): the reference Encoder, quant_conv and
    DiagonalGaussianDistribution.mode()."""

    def __init__(self, enc_sd, enc_cfg, quant_w, quant_b):
        super().__init__()
        self.enc = ref_shim.build_ref_encoder(enc_cfg)
        self.enc.load_state_dict(enc_sd, strict=True)
        self.qw, self.qb = quant_w, quant_b

    def encode(self, x):
        from sgm.modules.distributions.distributions import DiagonalGaussianDistribution
        return DiagonalGaussianDistribution(torch.nn.functional.conv2d(self.enc(x), self.qw, self.qb)).mode()


def reference_classes(sd, cfg):
    """The reference's embedder / conditioner classes, executed against stub open_clip / kornia, registered as the module
    `sgm.modules.encoders.modules` so that `target:` strings resolve to them."""
    ref_shim.install()
    from einops import rearrange, repeat
    from sgm.modules.diffusionmodules.util import timestep_embedding
    oc, ko = stub_packages(sd, cfg)

    class Timestep(nn.Module):                # openaimodel.py:466-472
        def __init__(self, dim):
            super().__init__()
            self.dim = dim

        def forward(self, t):
            return timestep_embedding(t, self.dim)

    path = os.path.join(ref_shim.REF, "sgm", "modules", "encoders", "modules.py")
    tree = ast.parse(open(path).read())
    want = ("AbstractEmbModel", "GeneralConditioner", "FrozenOpenCLIPImageEmbedder", "FrozenOpenCLIPImagePredictionEmbedder",
            "VideoPredictionEmbedderWithEncoder", "ConcatTimestepEmbedderND", "SphericalEmbedder")
    body = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name in want]
    assert len(body) == len(want)
    from sgm.util import append_dims, default, expand_dims_like
    mod = types.ModuleType("sgm.modules.encoders.modules")
    mod.__dict__.update({"torch": torch, "nn": nn, "np": np, "math": math, "nullcontext": nullcontext,
                         "Union": typing.Union, "List": typing.List, "Dict": typing.Dict, "Optional": typing.Optional,
                         "Tuple": typing.Tuple, "ListConfig": list, "instantiate_from_config": instantiate_from_config,
                         "disabled_train": lambda self, mode=True: self, "count_params": lambda m, verbose=False: 0,
                         "print": lambda *a, **k: None, "open_clip": oc, "kornia": ko, "autocast": lambda f: f,
                         "default": default, "expand_dims_like": expand_dims_like, "append_dims": append_dims,
                         "rearrange": rearrange, "repeat": repeat, "Timestep": Timestep})
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), mod.__dict__)
    pkg = types.ModuleType("sgm.modules.encoders")
    pkg.__path__ = []
    sys.modules["sgm.modules.encoders"], sys.modules["sgm.modules.encoders.modules"] = pkg, mod
    return mod


def maxrel(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


def pin_tower(tag, cfg, sizes):
    sd = visual_state(cfg)
    R = reference_classes(sd, cfg)
    emb = R.FrozenOpenCLIPImageEmbedder(freeze=True)
    out = {"cfg": cfg, "sizes": sizes, "pre_stride": PRE_STRIDE}
    for n, H, W in sizes:
        x = frames(n, H, W, frame_seed(n, H, W))
        z = emb(x)
        pre = emb.preprocess(x)
        e = maxrel(CO.clip_image_embed(sd, cfg, x), z)
        print(f"[clip {tag}] {n}x{H}x{W}: reference wrapper vs oracle {e:.1e}, |z| {z.norm():.3e}")
        assert e == 0.0 and z.shape == (n, cfg["embed"])
        out[f"z_{n}x{H}x{W}"] = z.clone()
        out[f"pre_{n}x{H}x{W}"] = pre[:, :, ::PRE_STRIDE, ::PRE_STRIDE].clone()
    torch.save(out, os.path.join(GOLD, f"clip_{tag}.pt"))


def pin_conditioning(tag, spherical):
    """GeneralConditioner.get_unconditional_conditioning over the GCD embedder list (tiny tower and encoder), as
    DiffusionEngine.sample_video calls it (models/diffusion.py:522-524)."""
    cfg, enc_cfg = clip.VIT_TINY, dict(spec.VAE_ENCODER_TINY)
    sd = visual_state(cfg, seed=1)
    R = reference_classes(sd, cfg)
    enc_sd = weights.seeded_state(spec.encoder_param_shapes(enc_cfg), seed=2)
    g = torch.Generator().manual_seed(55)
    zc = enc_cfg["z_channels"]
    qw, qb = torch.randn(2 * zc, 2 * zc, 1, 1, generator=g) * 0.4, torch.randn(2 * zc, generator=g) * 0.1
    sph_w, sph_b = torch.randn(128, 13, generator=g) * 0.3, torch.randn(128, generator=g) * 0.1
    sys.modules["_gcd_pin_ae"] = types.SimpleNamespace(AE=lambda **kw: _RefAEModeOnly(enc_sd, enc_cfg, qw, qb))
    emb_models = [
        {"input_key": "cond_frames_without_noise", "is_trainable": False,
         "target": "sgm.modules.encoders.modules.FrozenOpenCLIPImagePredictionEmbedder",
         "params": {"n_cond_frames": 1, "n_copies": 1, "open_clip_embedding_config": {
             "target": "sgm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder", "params": {"freeze": True}}}},
        {"input_key": "fps_id", "is_trainable": False, "target": "sgm.modules.encoders.modules.ConcatTimestepEmbedderND",
         "params": {"outdim": 256}},
        {"input_key": "motion_bucket_id", "is_trainable": True, "target": "sgm.modules.encoders.modules.ConcatTimestepEmbedderND",
         "params": {"outdim": 256}},
        {"input_key": "cond_frames", "is_trainable": False, "target": "sgm.modules.encoders.modules.VideoPredictionEmbedderWithEncoder",
         "params": {"disable_encoder_autocast": True, "en_and_decode_n_samples_a_time": 2, "n_cond_frames": 1, "n_copies": 1,
                    "is_ae": True, "encoder_config": {"target": "_gcd_pin_ae.AE"}}},
        {"input_key": "cond_aug", "is_trainable": False, "target": "sgm.modules.encoders.modules.ConcatTimestepEmbedderND",
         "params": {"outdim": 256}}]
    if spherical:
        emb_models.append({"input_key": "scaled_relative_angles", "is_trainable": True,
                           "target": "sgm.modules.encoders.modules.SphericalEmbedder", "params": {"embed_dim": 128}})
    cond = R.GeneralConditioner(emb_models)
    if spherical:
        cond.embedders[5].proj.weight.data.copy_(sph_w)
        cond.embedders[5].proj.bias.data.copy_(sph_b)
    n, (H, W) = COND_FRAMES, COND_HW
    batch = {"cond_frames_without_noise": frames(n, H, W, 71), "fps_id": torch.tensor([6.0, 6.0]),
             "motion_bucket_id": torch.tensor([127.0, 127.0]), "cond_aug": torch.tensor([0.02, 0.02])}
    batch["cond_frames"] = batch["cond_frames_without_noise"] + 0.02 * torch.randn(n, 3, H, W, generator=g)
    if spherical:
        batch["scaled_relative_angles"] = torch.tensor([[0.3, -0.2, 1.1], [-1.2, 0.4, 0.9]])
    c, uc = cond.get_unconditional_conditioning(batch, batch_uc=batch,
                                                force_uc_zero_embeddings=["cond_frames", "cond_frames_without_noise"])
    print(f"[conditioning {tag}] " + ", ".join(f"{k} {tuple(v.shape)}" for k, v in c.items()))
    assert c["vector"].shape[1] == (896 if spherical else 768)
    torch.save({"vit_cfg": cfg, "vit_seed": 1, "enc_cfg": enc_cfg, "enc_seed": 2, "quant_w": qw, "quant_b": qb,
                "sph_w": sph_w, "sph_b": sph_b, "batch": batch, "c": c, "uc": uc,
                "note": "open_clip / kornia arithmetic restated in oracle/clip_oracle.py; everything else is reference code"},
               os.path.join(GOLD, f"cond_{tag}.pt"))


def dump_cond_ae_decoder_keys():
    """Keys and shapes of the half of GCD's conditioning autoencoder (AutoencodingEngineLegacy, models/autoencoder.py:459-510,
    ddconfig of infer_kubric.yaml:83-94) that VideoPredictionEmbedderWithEncoder never runs: the reference `Decoder` and
    `post_quant_conv`. A GCD checkpoint carries them under `conditioner.embedders.3.encoder.`."""
    import json
    ref_shim.install()
    from sgm.modules.diffusionmodules.model import Decoder
    dd = dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128,
              ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0)
    with torch.device("meta"):
        dec = Decoder(**dd)
    keys = {"decoder." + k: list(v.shape) for k, v in dec.state_dict().items()}
    keys.update({"post_quant_conv.weight": [4, 4, 1, 1], "post_quant_conv.bias": [4]})
    json.dump(keys, open(os.path.join(GOLD, "cond_ae_decoder_keys.json"), "w"), indent=0, sort_keys=True)
    print(f"[conditioning autoencoder] {len(keys)} decoder-half keys")


if __name__ == "__main__":
    os.makedirs(GOLD, exist_ok=True)
    torch.manual_seed(0)
    dump_cond_ae_decoder_keys()
    pin_tower("tiny", clip.VIT_TINY, SIZES_TINY)
    pin_conditioning("kubric_tiny", spherical=True)
    pin_conditioning("pardom_tiny", spherical=False)
    if "--full" in sys.argv:
        pin_tower("full", clip.VIT_H14, SIZES_FULL)
