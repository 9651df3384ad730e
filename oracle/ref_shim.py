"""Imports the reference's own hot-path modules from a checkout of basilevh/gcd (TEST INFRASTRUCTURE: only the scripts that
write tests/golden/ use it; the tests themselves read the stored goldens). Point GCD_REFERENCE at the checkout's `gcd-model`
directory.

`import sgm` fails upstream (needs pytorch_lightning / omegaconf / open_clip / kornia, absent here — SURVEY.md §8(c)),
so empty package shells named `sgm`, `sgm.modules`, `sgm.models` are pre-registered with __path__ pointing at the
reference tree (their __init__.py never runs) plus a stub `omegaconf` (type hints only, sampling.py:9).
"""
import os
import sys
import types

REF = os.environ.get("GCD_REFERENCE", "")


def available():
    return bool(REF) and os.path.isdir(os.path.join(REF, "sgm"))


def install():
    if "sgm" in sys.modules and getattr(sys.modules["sgm"], "_gcd_shim", False):
        return
    if not available():
        raise RuntimeError("reference tree not found: set GCD_REFERENCE to the gcd-model directory of a basilevh/gcd checkout")
    for name, sub in (("sgm", "sgm"), ("sgm.modules", "sgm/modules"), ("sgm.models", "sgm/models"),
                      ("sgm.modules.autoencoding", "sgm/modules/autoencoding"),
                      ("sgm.modules.diffusionmodules", "sgm/modules/diffusionmodules")):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF, sub)]
        m._gcd_shim = True
        sys.modules[name] = m
    if "omegaconf" not in sys.modules:
        oc = types.ModuleType("omegaconf")
        oc.ListConfig = list
        oc.OmegaConf = type("OmegaConf", (), {})
        oc.DictConfig = dict
        sys.modules["omegaconf"] = oc


def build_ref_unet(cfg):
    """Reference VideoUNet (video_model.py:84) on CPU with *uninitialised* storage; caller loads a state dict."""
    install()
    import torch
    from sgm.modules.diffusionmodules.video_model import VideoUNet
    kw = dict(adm_in_channels=cfg["adm_in_channels"], num_classes="sequential", use_checkpoint=False,
              in_channels=cfg["in_channels"], out_channels=cfg["out_channels"], model_channels=cfg["model_channels"],
              attention_resolutions=cfg["attention_resolutions"], num_res_blocks=cfg["num_res_blocks"],
              channel_mult=cfg["channel_mult"], num_head_channels=cfg["num_head_channels"],
              use_linear_in_transformer=True, transformer_depth=cfg["transformer_depth"],
              context_dim=cfg["context_dim"], spatial_transformer_attn_type="softmax", extra_ff_mix_layer=True,
              use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1],
              aux_emb_dim=cfg["aux_emb_dim"], aux_zero_init=False)
    with torch.device("meta"):
        net = VideoUNet(**kw)
    net = net.to_empty(device="cpu")
    return net.eval()


def build_ref_decoder(cfg):
    install()
    import torch
    from sgm.modules.autoencoding.temporal_ae import VideoDecoder
    kw = dict(attn_type="vanilla", double_z=True, z_channels=cfg["z_channels"], resolution=256, in_channels=3,
              out_ch=cfg["out_ch"], ch=cfg["ch"], ch_mult=cfg["ch_mult"], num_res_blocks=cfg["num_res_blocks"],
              attn_resolutions=[], dropout=0.0, video_kernel_size=[3, 1, 1])
    with torch.device("meta"):
        dec = VideoDecoder(**kw)
    return dec.to_empty(device="cpu").eval()


def build_ref_encoder(cfg):
    """Reference VAE Encoder (diffusionmodules/model.py:487) on CPU with uninitialised storage."""
    install()
    import torch
    from sgm.modules.diffusionmodules.model import Encoder
    kw = dict(attn_type="vanilla", double_z=cfg.get("double_z", True), z_channels=cfg["z_channels"], resolution=256,
              in_channels=cfg["in_channels"], out_ch=3, ch=cfg["ch"], ch_mult=cfg["ch_mult"],
              num_res_blocks=cfg["num_res_blocks"], attn_resolutions=[], dropout=0.0)
    with torch.device("meta"):
        enc = Encoder(**kw)
    return enc.to_empty(device="cpu").eval()


def ref_embedder_classes():
    """The reference's own ConcatTimestepEmbedderND / SphericalEmbedder classes. `sgm/modules/encoders/modules.py` cannot be
    imported here (open_clip, kornia, transformers' CLIP/T5 at module top), so the three class definitions are cut out of the
    reference source with `ast` and executed against the real `Timestep` (openaimodel.py:466) — reference code runs, nothing
    is copied into this repository."""
    install()
    import ast
    import torch
    import torch.nn as nn
    from einops import rearrange
    from sgm.modules.diffusionmodules.util import timestep_embedding

    class Timestep(nn.Module):                 # openaimodel.py:466-472 (importing openaimodel needs the attention stack; 3 lines)
        def __init__(self, dim):
            super().__init__()
            self.dim = dim

        def forward(self, t):
            return timestep_embedding(t, self.dim)

    path = os.path.join(REF, "sgm", "modules", "encoders", "modules.py")
    tree = ast.parse(open(path).read())
    want = ("AbstractEmbModel", "SphericalEmbedder", "ConcatTimestepEmbedderND")
    body = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name in want]
    assert len(body) == 3
    ns = {"torch": torch, "nn": nn, "rearrange": rearrange, "Timestep": Timestep, "Union": __import__("typing").Union}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns["ConcatTimestepEmbedderND"], ns["SphericalEmbedder"]


def conditioner_classes():
    """The reference's AbstractEmbModel and GeneralConditioner. Their module cannot be imported here (open_clip / kornia), so
    the two class definitions are cut out of the reference source with `ast` and executed."""
    install()
    import ast
    import typing
    import torch
    import torch.nn as nn
    from gcd_b200.sampling import instantiate_from_config
    path = os.path.join(REF, "sgm", "modules", "encoders", "modules.py")
    tree = ast.parse(open(path).read())
    body = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name in ("AbstractEmbModel", "GeneralConditioner")]
    assert len(body) == 2
    ns = {"torch": torch, "nn": nn, "Union": typing.Union, "List": typing.List, "Dict": typing.Dict, "Optional": typing.Optional,
          "ListConfig": list, "instantiate_from_config": instantiate_from_config, "disabled_train": lambda self, mode=True: self,
          "count_params": lambda m, verbose=False: 0, "print": lambda *a, **k: None}
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), ns)
    return ns
