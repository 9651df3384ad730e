"""The two small vector embedders of the GCD conditioner (SURVEY.md §8(f) rank 1), as drop-in `target:`s:

* `ConcatTimestepEmbedderND` (encoders/modules.py:1000-1016): every scalar of x[b, d] -> sinusoidal embedding of `outdim`
  (util.py:207-231), concatenated to [b, d*outdim]. Used for fps_id / motion_bucket_id / cond_aug (infer_kubric.yaml:57-66,98-103).
* `SphericalEmbedder` (encoders/modules.py:247-287): (azimuth, elevation, radius) -> 13 trigonometric features -> Linear(13, dim).

Both run as one CUDA kernel each from libgcd_b200.so; like the rest of the package there is no CPU path. The properties the
reference's GeneralConditioner reads from AbstractEmbModel (is_trainable / ucg_rate / input_key, encoders/modules.py:40-81) exist.
"""
import torch
import torch.nn as nn

from . import clip, ops
from .engine import EngineCache, need_option, reference_base, register_param_tree

# The reference GeneralConditioner asserts `isinstance(embedder, AbstractEmbModel)` (encoders/modules.py:93-96): when `sgm`
# imports, the embedders derive from its AbstractEmbModel so a YAML `target:` swap passes that gate; standalone, from a plain
# nn.Module carrying the same three attributes (encoders/modules.py:40-81).
_RefBase = reference_base("sgm.modules.encoders.modules", "AbstractEmbModel")


class _EmbBase(_RefBase):
    def __init__(self):
        super().__init__()
        if _RefBase is nn.Module:
            self.is_trainable, self.ucg_rate, self.input_key = None, None, None

    @staticmethod
    def _need_cuda(x, who):
        if not x.is_cuda:
            raise RuntimeError(f"gcd_b200.{who} runs on CUDA (sm_90a) only; there is no CPU path")


class ConcatTimestepEmbedderND(_EmbBase):
    def __init__(self, outdim):
        super().__init__()
        if outdim % 2:
            raise NotImplementedError("gcd_b200.ConcatTimestepEmbedderND: odd outdim is not built (GCD uses 256)")
        self.outdim = outdim

    @torch.no_grad()
    def forward(self, x):
        self._need_cuda(x, "ConcatTimestepEmbedderND")
        if x.ndim == 1:
            x = x[:, None]
        assert x.ndim == 2
        b, dims = x.shape
        emb = torch.empty(b * dims, self.outdim, device=x.device, dtype=torch.float32)
        ops.timestep_embedding(x.reshape(-1).to(torch.float32).contiguous(), self.outdim, out_f32=emb)
        return emb.view(b, dims * self.outdim)


class SphericalEmbedder(_EmbBase):
    def __init__(self, embed_dim=128, zero_init=False):
        super().__init__()
        self.proj = nn.Linear(13, embed_dim)
        if zero_init:
            self.proj.weight.data.zero_()
            self.proj.bias.data.zero_()

    @torch.no_grad()
    def forward(self, x):
        self._need_cuda(x, "SphericalEmbedder")
        assert x.shape[-1] == 3
        lead = x.shape[:-1]
        xf = x.reshape(-1, 3).to(torch.float32).contiguous()
        out = torch.empty(xf.shape[0], self.proj.out_features, device=x.device, dtype=torch.float32)
        ops.spherical_embed(xf, self.proj.weight.detach().to(torch.float32).contiguous(),
                            self.proj.bias.detach().to(torch.float32).contiguous(), out)
        return out.view(*lead, -1)


class FrozenOpenCLIPImageEmbedder(_EmbBase):
    """Drop-in for the conditioner's image tower (encoders/modules.py:653-815; GCD: infer_kubric.yaml:51-54): frames
    [n, 3, H, W] in [-1, 1] -> pooled, projected OpenCLIP ViT-H/14 embeddings [n, 1024] float32 (gcd_b200/clip.py).

    The module tree is the reference's `self.model` after `del model.transformer`: `model.visual.*` plus the text-side tensors
    that stay in the state dict, so a GCD checkpoint's `conditioner.embedders.0.open_clip.model.*` loads with strict=False and
    nothing left over. Nothing is downloaded: `version` is accepted and ignored, the weights come from the checkpoint."""

    def __init__(self, arch="ViT-H-14", version="laion2b_s32b_b79k", device="cuda", max_length=77, freeze=True, antialias=True,
                 ucg_rate=0.0, unsqueeze_dim=False, repeat_to_max_len=False, num_image_crops=0, output_tokens=False,
                 init_device=None, vit_cfg=None):
        super().__init__()
        need = need_option("FrozenOpenCLIPImageEmbedder")
        need(arch == "ViT-H-14", f"arch={arch!r}")
        need(num_image_crops == 0, "num_image_crops > 0")
        need(not output_tokens, "output_tokens=True")
        need(not repeat_to_max_len, "repeat_to_max_len=True")
        need(not ucg_rate, "ucg_rate > 0")
        need(antialias, "antialias=False")
        self.vit_cfg = dict(vit_cfg or clip.VIT_H14)              # vit_cfg: a smaller tower for tests (same 80-wide heads)
        self.model = nn.Module()
        self.model.add_module("visual", nn.Module())
        register_param_tree(self.model.visual, clip.visual_param_shapes(self.vit_cfg))
        if vit_cfg is None:
            register_param_tree(self.model, clip.TEXT_LEFTOVERS_H14)
        self.max_crops, self.max_length, self.device = num_image_crops, max_length, device
        self.antialias, self.unsqueeze_dim, self.output_tokens = antialias, unsqueeze_dim, output_tokens
        self.ucg_rate = ucg_rate
        if freeze:
            for p in self.parameters():
                p.requires_grad = False
        self._engines = EngineCache()

    def engine(self, device):
        visual = self.model.visual
        return self._engines.get(visual, device, lambda: clip.ClipEngine(self.vit_cfg, visual.state_dict(), device))

    @torch.no_grad()
    def forward(self, image, no_dropout=False):
        self._need_cuda(image, "FrozenOpenCLIPImageEmbedder")
        if image.dim() != 4 or image.shape[1] != 3:
            raise ValueError("FrozenOpenCLIPImageEmbedder expects [n, 3, H, W] frames")
        z = self.engine(image.device).forward(image).to(image.dtype)
        return z[:, None, :] if self.unsqueeze_dim else z

    def encode(self, image):
        return self(image)


class FrozenOpenCLIPImagePredictionEmbedder(_EmbBase):
    """encoders/modules.py:1117-1136: the image tower on every conditioning frame, "(b t) d -> b t d" over n_cond_frames, then
    repeated n_copies times -> the `crossattn` conditioning [b*n_copies, n_cond_frames, 1024]."""

    def __init__(self, open_clip_embedding_config, n_cond_frames, n_copies):
        super().__init__()
        from .sampling import instantiate_from_config
        self.n_cond_frames, self.n_copies = n_cond_frames, n_copies
        self.open_clip = instantiate_from_config(_local_target(open_clip_embedding_config))

    def forward(self, vid):
        z = self.open_clip(vid)
        b = z.shape[0] // self.n_cond_frames
        z = z.reshape(b, self.n_cond_frames, z.shape[-1])
        return z.repeat_interleave(self.n_copies, dim=0)


_LOCAL = {"sgm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder": "gcd_b200.embedders.FrozenOpenCLIPImageEmbedder"}


def _local_target(cfg):
    """The inner `target:` of the GCD configs names the reference class; it resolves to the one here (no open_clip)."""
    cfg = dict(cfg)
    cfg["target"] = _LOCAL.get(cfg["target"], cfg["target"])
    return cfg


class AutoencoderKLModeOnly(nn.Module):
    """The conditioner-side autoencoder of GCD (models/autoencoder.py:627-640, infer_kubric.yaml:77-96) as far as
    VideoPredictionEmbedderWithEncoder uses it: `encoder` (gcd_b200.vae.Encoder) and `quant_conv`; encode() is the mode of the
    diagonal Gaussian. The decoder half of the reference module is never run, so its checkpoint keys stay unexpected."""

    def __init__(self, embed_dim, ddconfig, **ignore):
        super().__init__()
        from .vae import Encoder
        self.encoder = Encoder(**ddconfig)
        zc = ddconfig["z_channels"]
        if not ddconfig.get("double_z", True) or embed_dim != zc:
            raise NotImplementedError("gcd_b200.AutoencoderKLModeOnly: only double_z with embed_dim == z_channels is built")
        self.quant_conv = nn.Conv2d(2 * zc, 2 * embed_dim, 1)

    @torch.no_grad()
    def encode(self, x, scale_factor=1.0):
        return self.encoder.encode_mode(x, self.quant_conv.weight, self.quant_conv.bias, scale_factor)


class VideoPredictionEmbedderWithEncoder(_EmbBase):
    """encoders/modules.py:1039-1114 without noise augmentation: scale_factor * mode(encode(frames)), "(b t) c h w ->
    b () (t c) h w" over n_cond_frames, repeated n_copies times -> the `concat` conditioning. Splitting the frames into chunks of
    `en_and_decode_n_samples_a_time` does not change the result (the encoder is per frame), so they are encoded at once."""

    def __init__(self, n_cond_frames, n_copies, encoder_config, sigma_sampler_config=None, sigma_cond_config=None, is_ae=False,
                 scale_factor=1.0, disable_encoder_autocast=False, en_and_decode_n_samples_a_time=None):
        super().__init__()
        if sigma_sampler_config is not None or sigma_cond_config is not None or not is_ae:
            raise NotImplementedError("gcd_b200.VideoPredictionEmbedderWithEncoder: noise augmentation / non-AE encoders are not "
                                      "built (GCD sets neither)")
        from .sampling import instantiate_from_config
        self.n_cond_frames, self.n_copies, self.scale_factor = n_cond_frames, n_copies, scale_factor
        self.encoder = instantiate_from_config(_local_target(encoder_config))

    @torch.no_grad()
    def forward(self, vid):
        self._need_cuda(vid, "VideoPredictionEmbedderWithEncoder")
        z = self.encoder.encode(vid, self.scale_factor)
        bt, c, h, w = z.shape
        z = z.reshape(bt // self.n_cond_frames, self.n_cond_frames * c, h, w)
        return z.repeat_interleave(self.n_copies, dim=0)


_LOCAL.update({"sgm.modules.encoders.modules.FrozenOpenCLIPImagePredictionEmbedder":
               "gcd_b200.embedders.FrozenOpenCLIPImagePredictionEmbedder",
               "sgm.modules.encoders.modules.ConcatTimestepEmbedderND": "gcd_b200.embedders.ConcatTimestepEmbedderND",
               "sgm.modules.encoders.modules.VideoPredictionEmbedderWithEncoder":
               "gcd_b200.embedders.VideoPredictionEmbedderWithEncoder",
               "sgm.models.autoencoder.AutoencoderKLModeOnly": "gcd_b200.embedders.AutoencoderKLModeOnly",
               "sgm.modules.encoders.modules.SphericalEmbedder": "gcd_b200.embedders.SphericalEmbedder"})


def gcd_conditioner_config(spherical=True, vit_cfg=None, enc_cfg=None):
    """`conditioner_config.params.emb_models` of infer_kubric.yaml:45-110 (spherical=True) / infer_pardom.yaml with this
    package's targets. vit_cfg / enc_cfg: smaller towers for tests."""
    from . import spec
    enc = dict(enc_cfg or spec.VAE_ENCODER)
    clip_params = {"freeze": True} if vit_cfg is None else {"freeze": True, "vit_cfg": dict(vit_cfg)}
    ddconfig = {"attn_type": "vanilla-xformers", "double_z": True, "z_channels": enc["z_channels"], "resolution": 256,
                "in_channels": enc["in_channels"], "out_ch": 3, "ch": enc["ch"], "ch_mult": list(enc["ch_mult"]),
                "num_res_blocks": enc["num_res_blocks"], "attn_resolutions": [], "dropout": 0.0}
    ts = lambda key, trainable=False: {"input_key": key, "is_trainable": trainable,
                                       "target": "gcd_b200.embedders.ConcatTimestepEmbedderND", "params": {"outdim": 256}}
    cfg = [{"input_key": "cond_frames_without_noise", "is_trainable": False,
            "target": "gcd_b200.embedders.FrozenOpenCLIPImagePredictionEmbedder",
            "params": {"n_cond_frames": 1, "n_copies": 1, "open_clip_embedding_config": {
                "target": "gcd_b200.embedders.FrozenOpenCLIPImageEmbedder", "params": clip_params}}},
           ts("fps_id"), ts("motion_bucket_id", True),
           {"input_key": "cond_frames", "is_trainable": False, "target": "gcd_b200.embedders.VideoPredictionEmbedderWithEncoder",
            "params": {"disable_encoder_autocast": True, "en_and_decode_n_samples_a_time": 2, "n_cond_frames": 1, "n_copies": 1,
                       "is_ae": True, "encoder_config": {"target": "gcd_b200.embedders.AutoencoderKLModeOnly",
                                                         "params": {"embed_dim": enc["z_channels"], "ddconfig": ddconfig}}}},
           ts("cond_aug")]
    if spherical:
        cfg.append({"input_key": "scaled_relative_angles", "is_trainable": True, "target": "gcd_b200.embedders.SphericalEmbedder",
                    "params": {"embed_dim": 128, "zero_init": False}})
    return cfg


def build_embedders(emb_models):
    """The embedder modules of a conditioner config, in config order (what GeneralConditioner.embedders holds)."""
    from .sampling import instantiate_from_config
    return [instantiate_from_config(_local_target(e)) for e in emb_models]
