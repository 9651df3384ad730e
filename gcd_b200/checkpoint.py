"""Checkpoint ingest for the drop-in modules (SURVEY.md §8(f) rank 3, first slice): what `DiffusionEngine.init_from_ckpt`
(models/diffusion.py:191-219) does for the tensors of the hot path.

The reference loads `.ckpt` (`torch.load(...)["state_dict"]`) or `.safetensors` files whose keys carry the DiffusionEngine's module
prefixes and calls `self.load_state_dict(sd, strict=False)` — a renamed key would be skipped SILENTLY. `HotPathRoot` reproduces
that module tree for the parts this package replaces, so the same call works and the (missing, unexpected) lists can be checked:

    model.diffusion_model.*                      gcd_b200.unet.VideoUNet            (OpenAIWrapper.diffusion_model, wrappers.py:10-21)
    first_stage_model.decoder.*                  gcd_b200.vae.VideoDecoder          (autoencoder.py `self.decoder`)
    first_stage_model.encoder.*                  gcd_b200.vae.Encoder (optional)
    first_stage_model.quant_conv.*               1x1 conv of AutoencoderKL (folded into Encoder.encode_mode)
    model_ema.*                                  LitEma shadows of `model` (modules/ema.py: name with the dots removed)
    conditioner.embedders.<i>.*                  gcd_b200.embedders (optional, HotPathRoot(conditioner=...))

Host-side plumbing only: no kernels involved; the modules repack their weights for the CUDA engines on the next forward
(gcd_b200.engine.weights_key).
"""
import os

import torch
import torch.nn as nn

from . import sampling


def read_state_dict(path):
    """The reference's file handling (models/diffusion.py:193-199)."""
    assert os.path.exists(path) and os.path.isfile(path), path
    if path.endswith("ckpt"):
        return torch.load(path, map_location="cpu", weights_only=False)["state_dict"]
    if path.endswith("safetensors"):
        from safetensors.torch import load_file
        return load_file(path)
    raise NotImplementedError(f"unsupported checkpoint format: {path}")


class _FirstStage(nn.Module):
    def __init__(self, decoder, encoder=None, z_channels=4):
        super().__init__()
        self.decoder = decoder
        if encoder is not None:
            self.encoder = encoder
            self.quant_conv = nn.Conv2d(2 * z_channels, 2 * z_channels, 1)       # autoencoder.py AutoencoderKL.quant_conv


class HotPathRoot(nn.Module):
    """Module tree with the DiffusionEngine's attribute names for the replaced components (everything else in a checkpoint —
    conditioner, loss, optimizer — lands in `unexpected`, exactly like unknown keys do in the reference's strict=False load)."""

    def __init__(self, unet, decoder, encoder=None, conditioner=None):
        """`conditioner`: optional embedder modules in YAML order (gcd_b200.embedders.build_embedders), registered as
        `conditioner.embedders.<i>` — GeneralConditioner's attribute names — so the CLIP tower
        (`conditioner.embedders.0.open_clip.model.*`), the conditioning-frame encoder (`...3.encoder.{encoder,quant_conv}.*`)
        and the spherical embedder (`...5.proj.*`) load through the same call. The decoder half of that autoencoder
        (`...3.encoder.{decoder,post_quant_conv}.*`) has no module here and stays in `unexpected`."""
        super().__init__()
        self.model = sampling.OpenAIWrapper(unet)
        self.first_stage_model = _FirstStage(decoder, encoder)
        if conditioner is not None:
            self.conditioner = nn.Module()
            self.conditioner.embedders = nn.ModuleList(list(conditioner))

    def init_from_ckpt(self, path, use_ema=False):
        """models/diffusion.py:191-219. Returns (missing, unexpected); with use_ema the `model_ema.*` shadows overwrite the
        UNet weights afterwards (what sampling under `ema_scope` uses, models/diffusion.py:278-292)."""
        sd = read_state_dict(path)
        missing, unexpected = self.load_state_dict(sd, strict=False)
        if use_ema:
            n = apply_ema(sd, self.model)
            if n == 0:
                raise KeyError("use_ema=True but the checkpoint holds no model_ema.* shadows")
            unexpected = [k for k in unexpected if not k.startswith("model_ema.")]
        return list(missing), list(unexpected)


def ema_key(param_name):
    """LitEma buffer name of a parameter (modules/ema.py:19-24: '.' is not allowed in buffer names)."""
    return param_name.replace(".", "")


@torch.no_grad()
def apply_ema(sd, model, prefix="model_ema."):
    """Copies the EMA shadows of `sd` into `model`'s parameters (LitEma.copy_to, modules/ema.py:52-60). Returns the number of
    tensors copied; raises if a parameter with a shadow in the file has a different shape."""
    n = 0
    for name, p in model.named_parameters():
        k = prefix + ema_key(name)
        if k in sd:
            if tuple(sd[k].shape) != tuple(p.shape):
                raise ValueError(f"EMA shadow {k}: shape {tuple(sd[k].shape)} != parameter {tuple(p.shape)}")
            p.data.copy_(sd[k])
            n += 1
    return n
