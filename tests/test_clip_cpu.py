"""CPU tests of the conditioner's image tower: module tree / state-dict contract of FrozenOpenCLIPImageEmbedder, rejected
options, the GCD embedder list through instantiate_from_config, checkpoint ingest through HotPathRoot(conditioner=...), and
the fp32 oracle against the stored goldens."""
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _meta(fn):
    with torch.device("meta"):
        return fn()


def test_vit_h14_visual_state_dict_keys_and_shapes():
    from gcd_b200.embedders import FrozenOpenCLIPImageEmbedder
    emb = _meta(lambda: FrozenOpenCLIPImageEmbedder())
    sd = {k: tuple(v.shape) for k, v in emb.state_dict().items()}
    expected = {"model.visual.conv1.weight": (1280, 3, 14, 14), "model.visual.class_embedding": (1280,),
                "model.visual.positional_embedding": (257, 1280), "model.visual.ln_pre.weight": (1280,),
                "model.visual.ln_pre.bias": (1280,), "model.visual.ln_post.weight": (1280,),
                "model.visual.ln_post.bias": (1280,), "model.visual.proj": (1280, 1024),
                "model.token_embedding.weight": (49408, 1024), "model.positional_embedding": (77, 1024),
                "model.ln_final.weight": (1024,), "model.ln_final.bias": (1024,), "model.text_projection": (1024, 1024),
                "model.logit_scale": ()}
    for i in range(32):
        b = f"model.visual.transformer.resblocks.{i}."
        expected.update({b + "ln_1.weight": (1280,), b + "ln_1.bias": (1280,),
                         b + "attn.in_proj_weight": (3840, 1280), b + "attn.in_proj_bias": (3840,),
                         b + "attn.out_proj.weight": (1280, 1280), b + "attn.out_proj.bias": (1280,),
                         b + "ln_2.weight": (1280,), b + "ln_2.bias": (1280,),
                         b + "mlp.c_fc.weight": (5120, 1280), b + "mlp.c_fc.bias": (5120,),
                         b + "mlp.c_proj.weight": (1280, 5120), b + "mlp.c_proj.bias": (1280,)})
    assert sd == expected
    assert sum(torch.Size(s).numel() for k, s in expected.items() if k.startswith("model.visual.")) == 632_076_800
    assert not any(p.requires_grad for p in emb.parameters())                     # freeze=True


@pytest.mark.parametrize("kw", [dict(num_image_crops=1), dict(output_tokens=True), dict(repeat_to_max_len=True),
                                dict(ucg_rate=0.1), dict(arch="ViT-L-14"), dict(antialias=False)])
def test_unsupported_options_raise(kw):
    from gcd_b200.embedders import FrozenOpenCLIPImageEmbedder
    with pytest.raises(NotImplementedError):
        FrozenOpenCLIPImageEmbedder(**kw)


def test_vae_embedder_rejects_noise_augmentation():
    from gcd_b200.embedders import VideoPredictionEmbedderWithEncoder
    with pytest.raises(NotImplementedError):
        VideoPredictionEmbedderWithEncoder(1, 1, {"target": "torch.nn.Identity"}, sigma_sampler_config={"target": "x"}, is_ae=True)


def test_gcd_embedder_list_resolves_through_instantiate_from_config():
    from gcd_b200 import embedders as E
    from gcd_b200.clip import VIT_TINY
    from gcd_b200.spec import VAE_ENCODER_TINY
    for spherical in (True, False):
        cfg = E.gcd_conditioner_config(spherical=spherical, vit_cfg=VIT_TINY, enc_cfg=VAE_ENCODER_TINY)
        mods = E.build_embedders(cfg)
        names = [type(m).__name__ for m in mods]
        assert names == ["FrozenOpenCLIPImagePredictionEmbedder", "ConcatTimestepEmbedderND", "ConcatTimestepEmbedderND",
                         "VideoPredictionEmbedderWithEncoder", "ConcatTimestepEmbedderND"] + (["SphericalEmbedder"] if spherical else [])
        assert [c["input_key"] for c in cfg][:5] == ["cond_frames_without_noise", "fps_id", "motion_bucket_id", "cond_frames",
                                                     "cond_aug"]
        assert isinstance(mods[0].open_clip, E.FrozenOpenCLIPImageEmbedder)
    # the reference's own target strings resolve to the local classes (no open_clip import)
    inner = E._local_target({"target": "sgm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder"})
    assert inner["target"] == "gcd_b200.embedders.FrozenOpenCLIPImageEmbedder"


# The decoder half of GCD's conditioning autoencoder (AutoencodingEngineLegacy, models/autoencoder.py:459-510): the reference
# `Decoder` + `post_quant_conv` keys, dumped from the reference by oracle/pin_clip.py. They have no module here and must be exactly
# the `conditioner.` keys left in `unexpected`.
def _decoder_half_keys():
    import json
    with open(os.path.join(GOLD, "cond_ae_decoder_keys.json")) as f:
        keys = json.load(f)
    assert len(keys) == 140 and "decoder.conv_in.weight" in keys and "decoder.up.3.upsample.conv.weight" in keys
    return {f"conditioner.embedders.3.encoder.{k}": tuple(s) for k, s in keys.items()}


def test_hot_path_root_with_conditioner_round_trips_a_gcd_state_dict():
    from gcd_b200 import checkpoint, clip, embedders as E, spec
    from gcd_b200.unet import VideoUNet
    from gcd_b200.vae import Encoder, VideoDecoder
    enc_cfg = spec.VAE_ENCODER_TINY
    cond = E.build_embedders(E.gcd_conditioner_config(spherical=True, vit_cfg=clip.VIT_TINY, enc_cfg=enc_cfg))
    # without the argument: exactly the old module tree
    plain = checkpoint.HotPathRoot(VideoUNet(**spec.unet_ctor_kwargs(spec.UNET_TINY)),
                                   VideoDecoder(**spec.decoder_ctor_kwargs(spec.VAE_TINY)))
    assert not hasattr(plain, "conditioner")
    root = checkpoint.HotPathRoot(VideoUNet(**spec.unet_ctor_kwargs(spec.UNET_TINY)),
                                  VideoDecoder(**spec.decoder_ctor_kwargs(spec.VAE_TINY)),
                                  Encoder(**spec.encoder_ctor_kwargs(enc_cfg)), conditioner=cond)
    # a state dict with the key layout of a GCD checkpoint's conditioner (tiny widths)
    g = torch.Generator().manual_seed(0)
    file_sd = {}
    for k, v in plain.state_dict().items():
        file_sd[k] = torch.randn(v.shape, generator=g)
    vis = clip.visual_param_shapes(clip.VIT_TINY)
    pre = "conditioner.embedders.0.open_clip.model."
    file_sd.update({pre + "visual." + k: torch.randn(s, generator=g) for k, s in vis.items()})
    enc_keys = {f"conditioner.embedders.3.encoder.encoder.{k}": s for k, s in spec.encoder_param_shapes(enc_cfg).items()}
    enc_keys.update({"conditioner.embedders.3.encoder.quant_conv.weight": (8, 8, 1, 1),
                     "conditioner.embedders.3.encoder.quant_conv.bias": (8,),
                     "conditioner.embedders.5.proj.weight": (128, 13), "conditioner.embedders.5.proj.bias": (128,)})
    file_sd.update({k: torch.randn(s, generator=g) for k, s in enc_keys.items()})
    file_sd["first_stage_model.encoder.conv_in.weight"] = root.state_dict()["first_stage_model.encoder.conv_in.weight"] + 1
    file_sd.update({k: torch.zeros(s) for k, s in _decoder_half_keys().items()})
    missing, unexpected = root.load_state_dict(file_sd, strict=False)
    missing = [k for k in missing if not k.startswith("first_stage_model.encoder.") and not k.startswith("first_stage_model.quant_conv.")]
    assert missing == []
    assert not any(k.startswith(pre) for k in unexpected)
    assert sorted(k for k in unexpected if k.startswith("conditioner.")) == sorted(_decoder_half_keys())
    got = root.state_dict()
    for k in list(vis)[:5] + ["proj"]:
        assert torch.equal(got[pre + "visual." + k], file_sd[pre + "visual." + k])
    assert torch.equal(got["conditioner.embedders.5.proj.weight"], file_sd["conditioner.embedders.5.proj.weight"])
    assert torch.equal(got["conditioner.embedders.3.encoder.quant_conv.bias"], file_sd["conditioner.embedders.3.encoder.quant_conv.bias"])


def test_kornia_blur_taps():
    from gcd_b200.clip import kornia_blur_taps
    assert kornia_blur_taps(224, 224) is None and kornia_blur_taps(64, 96) is None
    tx, ty = kornia_blur_taps(576, 1024)             # factors 2.57 / 4.57 -> sigma 0.786 / 1.786 -> ks 3 / 7
    assert (tx.numel(), ty.numel()) == (7, 3)
    assert abs(tx.sum().item() - 1) < 1e-6 and torch.equal(tx, tx.flip(0))
    tx, ty = kornia_blur_taps(256, 384)              # factors 1.14 / 1.71 -> ks 3 / 3
    assert (tx.numel(), ty.numel()) == (3, 3)


@pytest.mark.parametrize("tag", ["tiny", "full"])
def test_oracle_reproduces_tower_goldens(tag):
    from gcd_b200 import synthetic
    from gcd_b200.clip import visual_param_shapes
    from oracle import clip_oracle as CO
    path = os.path.join(GOLD, f"clip_{tag}.pt")
    gold = torch.load(path)
    cfg = gold["cfg"]
    sd = synthetic.seeded_state(visual_param_shapes(cfg), seed=0)
    sizes = gold["sizes"] if tag == "tiny" else gold["sizes"][-1:]        # the full tower: the 2-frame case (CPU time)
    with torch.no_grad():
        for n, H, W in sizes:
            g = torch.Generator().manual_seed(1000 + n * 7 + H * 3 + W)
            x = torch.rand(n, 3, H, W, generator=g) * 2 - 1
            pre = CO.clip_preprocess(x)
            s = gold["pre_stride"]
            ref_pre, ref_z = gold[f"pre_{n}x{H}x{W}"], gold[f"z_{n}x{H}x{W}"]
            assert (pre[:, :, ::s, ::s] - ref_pre).abs().max().item() <= 1e-6
            z = CO.clip_visual_forward(sd, cfg, pre)
            assert ((z - ref_z).abs().max() / ref_z.abs().max()).item() < 1e-5
