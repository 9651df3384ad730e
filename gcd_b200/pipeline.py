"""Hot-path driver: what DiffusionEngine.sample_video does between conditioning and pixels
(models/diffusion.py:504-549): latent noise -> 25-step EDM/Euler sample (CFG) -> decode_first_stage (:233-251).
This is the public API bench.py measures end to end and the object tests/smoke drive; under gcd-model/ the same
classes are reached through `instantiate_from_config` (INTEGRATION.md)."""
import torch

from . import sampling, spec
from .unet import VideoUNet
from .vae import Encoder, VideoDecoder


class GCDHotPath:
    def __init__(self, unet_cfg=None, vae_cfg=None, num_steps=25, num_frames=14, max_scale=1.5, min_scale=1.0,
                 sigma_max=700.0, scale_factor=0.18215, device="cuda", unet=None, decoder=None):
        """`unet` / `decoder`: already loaded drop-in modules to share (a second sampler configuration over the same weights —
        e.g. 50 steps at max scale 2.5 next to the 25-step one — reuses their packed engines); built empty otherwise."""
        self.unet_cfg = dict(unet_cfg or spec.UNET_KUBRIC)
        self.vae_cfg = dict(vae_cfg or spec.VAE_DECODER)
        self.device = torch.device(device)
        self.T, self.scale_factor = num_frames, scale_factor
        self.unet = unet if unet is not None else VideoUNet(**spec.unet_ctor_kwargs(self.unet_cfg))
        self.decoder = decoder if decoder is not None else VideoDecoder(**spec.decoder_ctor_kwargs(self.vae_cfg))
        self.model = sampling.OpenAIWrapper(self.unet)
        self.denoiser = sampling.Denoiser({"target": "gcd_b200.sampling.VScalingWithEDMcNoise"})
        self.sampler = sampling.EulerEDMSampler(
            discretization_config={"target": "gcd_b200.sampling.EDMDiscretization", "params": {"sigma_max": sigma_max}},
            num_steps=num_steps,
            guider_config={"target": "gcd_b200.sampling.LinearPredictionGuider",
                           "params": {"num_frames": num_frames, "max_scale": max_scale, "min_scale": min_scale}},
            device=str(self.device))

    def load_state(self, unet_state, vae_state):
        self.unet.load_state_dict(unet_state, strict=True)
        self.decoder.load_state_dict(vae_state, strict=True)
        self.unet.to(self.device)
        self.decoder.to(self.device)
        return self

    def set_cfg_parallel(self, group):
        """Single-clip latency mode over a 2-rank group: see EulerEDMSampler.set_cfg_parallel."""
        self.sampler.set_cfg_parallel(group)
        return self

    def load_cond_encoder(self, encoder_state, quant_weight, quant_bias, enc_cfg=None):
        """Optional front-end (SURVEY.md §8(f) rank 1): the AutoencoderKLModeOnly that VideoPredictionEmbedderWithEncoder
        wraps (configs/infer_kubric.yaml:69-96). `encoder_state` uses the reference keys below `...encoder.encoder.`."""
        self.enc_cfg = dict(enc_cfg or spec.VAE_ENCODER)
        self.encoder = Encoder(**spec.encoder_ctor_kwargs(self.enc_cfg))
        self.encoder.load_state_dict(encoder_state, strict=True)
        self.encoder.to(self.device)
        self.quant = (quant_weight.to(self.device, torch.float32), quant_bias.to(self.device, torch.float32))
        return self

    @torch.no_grad()
    def encode_cond_frames(self, frames, n_cond_frames=1, n_copies=1, scale_factor=None):
        """VideoPredictionEmbedderWithEncoder.forward without noise augmentation (encoders/modules.py:1090-1109; the shipped
        configs set no sigma_sampler and n_cond_frames = n_copies = 1, infer_kubric.yaml:75-76): frames [B*T,3,H,W] in
        [-1,1] -> scale_factor * mode(encode), then "(b t) c h w -> b () (t c) h w" repeated n_copies times. The result is
        the `concat` conditioning the UNet wrapper appends to the noisy latents (wrappers.py:24). `scale_factor` defaults to
        the first-stage scale of this pipeline."""
        s = self.scale_factor if scale_factor is None else scale_factor
        z = self.encoder.encode_mode(frames.to(self.device, non_blocking=True), self.quant[0], self.quant[1], s)
        if n_cond_frames == 1 and n_copies == 1:
            return z
        bt, c, h, w = z.shape
        z = z.view(bt // n_cond_frames, 1, n_cond_frames * c, h, w)
        return z.expand(-1, n_copies, -1, -1, -1).reshape(-1, n_cond_frames * c, h, w)

    def load_clip(self, state, vit_cfg=None):
        """The conditioner's OpenCLIP ViT-H/14 image tower (gcd_b200.embedders.FrozenOpenCLIPImageEmbedder). `state`: its state
        dict, keys `model.visual.*` (the text-side leftovers of a checkpoint may be included). vit_cfg: a smaller tower."""
        from .embedders import FrozenOpenCLIPImageEmbedder
        clip = FrozenOpenCLIPImageEmbedder(vit_cfg=vit_cfg)
        missing, unexpected = clip.load_state_dict(state, strict=False)
        if missing or unexpected:
            raise KeyError(f"load_clip: missing {list(missing)[:5]}, unexpected {list(unexpected)[:5]}")
        self.clip = clip.to(self.device)
        return self

    def load_spherical(self, weight, bias):
        """SphericalEmbedder.proj of the Kubric conditioner (infer_kubric.yaml:105-110): weight [128, 13], bias [128]."""
        from .embedders import SphericalEmbedder
        self.spherical = SphericalEmbedder(weight.shape[0])
        self.spherical.proj.weight.data.copy_(weight)
        self.spherical.proj.bias.data.copy_(bias)
        self.spherical.to(self.device)
        return self

    @torch.no_grad()
    def condition(self, batch, cond_scale_factor=1.0):
        """(c, uc) of GeneralConditioner.get_unconditional_conditioning(batch, batch_uc=batch,
        force_uc_zero_embeddings=["cond_frames", "cond_frames_without_noise"]) (encoders/modules.py:84-208,
        models/diffusion.py:522-524) for the GCD embedder lists (infer_kubric.yaml:45-110, infer_pardom.yaml):
            crossattn  FrozenOpenCLIPImagePredictionEmbedder(cond_frames_without_noise)   [BT, 1, 1024]   (load_clip)
            vector     cat(fps_id, motion_bucket_id, cond_aug) timestep embeddings (256 each) [+ SphericalEmbedder(
                       scaled_relative_angles), 128, when the UNet takes an aux embedding]          [BT, 768 | 896]
            concat     VideoPredictionEmbedderWithEncoder(cond_frames)                  [BT, 4, H/8, W/8] (load_cond_encoder)
        uc: crossattn and concat zero, vector equal to c's. `cond_scale_factor` is that embedder's scale_factor (the configs
        leave the reference default 1.0). Noise augmentation of cond_frames is the caller's (eval_utils.py:224-225)."""
        from .embedders import ConcatTimestepEmbedderND
        dev = self.device
        get = lambda k: batch[k].to(dev, non_blocking=True)
        frames = get("cond_frames_without_noise")
        ca = self.clip(frames)[:, None, :]                          # n_cond_frames = n_copies = 1: "(b t) d -> b t d"
        ts = ConcatTimestepEmbedderND(256)
        vec = [ts(get(k)) for k in ("fps_id", "motion_bucket_id", "cond_aug")]
        if self.unet_cfg.get("aux_emb_dim", 0):
            if getattr(self, "spherical", None) is None:
                raise RuntimeError("condition: this UNet takes the spherical camera embedding; call load_spherical first")
            vec.append(self.spherical(get("scaled_relative_angles")))
        vector = torch.cat(vec, 1)
        concat = self.encode_cond_frames(get("cond_frames"), scale_factor=cond_scale_factor)
        c = {"crossattn": ca, "vector": vector, "concat": concat}
        uc = {"crossattn": torch.zeros_like(ca), "vector": vector.clone(), "concat": torch.zeros_like(concat)}
        return c, uc

    @torch.no_grad()
    def sample_latents(self, noise, c, uc, num_steps=None):
        """noise: float32 [B*T,4,h,w] on device (consumed in place, sampling.py:54). c/uc: dicts of device tensors."""
        BT = noise.shape[0]
        extra = dict(num_video_frames=self.T,
                     image_only_indicator=torch.zeros(2 * BT // self.T, self.T, device=noise.device))
        den = sampling.FusedDenoiser(self.denoiser, self.model, **extra)
        return self.sampler(den, noise, cond=c, uc=uc, num_steps=num_steps)

    @torch.no_grad()
    def decode_first_stage(self, z, decoding_t=None):
        """models/diffusion.py:233-251: z / scale_factor, chunks of `decoding_t` frames, fp32."""
        z = z / self.scale_factor
        n = decoding_t or self.T
        outs = [self.decoder(z[i:i + n], timesteps=min(n, z.shape[0] - i)) for i in range(0, z.shape[0], n)]
        return torch.cat(outs, 0)

    @torch.no_grad()
    def sample_video(self, noise, c, uc, num_steps=None, decode=True):
        """Returns (latents [B*T,4,h,w], frames [B*T,3,8h,8w] or None). Host tensors are copied to the device first
        (that copy is part of the end-to-end measurement in bench.py)."""
        dev = self.device
        noise = noise.to(dev, non_blocking=True)
        c = {k: v.to(dev, non_blocking=True) for k, v in c.items()}
        uc = {k: v.to(dev, non_blocking=True) for k, v in uc.items()}
        z = self.sample_latents(noise, c, uc, num_steps)
        frames = self.decode_first_stage(z) if decode else None
        return z, frames


def shard_clips(num_clips, rank, world):
    """Clip indices owned by `rank`: strided like the reference's per-GPU worker buckets
    (`examples[bucket_idx::num_buckets]`, scripts/test.py:1059-1084). Clips are independent (SURVEY.md §8(e))."""
    return list(range(num_clips))[rank::world]


def gather_clips(local, num_clips, rank, world, group=None):
    """All-gathers per-rank clip tensors (each [T, ...], same shape) back into clip order. The ONLY collective on the
    path (NCCL over NVLink on GPUs; gloo in the CPU tests). local: list of tensors for shard_clips(num_clips, rank, world)."""
    import torch.distributed as dist
    per = (num_clips + world - 1) // world
    proto = local[0]
    pad = [torch.zeros_like(proto) for _ in range(per - len(local))]
    mine = torch.stack(list(local) + pad)                       # [per, T, ...]
    bufs = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(bufs, mine, group=group)
    out = [None] * num_clips
    for r in range(world):
        for j, idx in enumerate(shard_clips(num_clips, r, world)):
            out[idx] = bufs[r][j]
    return out
