"""The two small vector embedders of the GCD conditioner (SURVEY.md §8(f) rank 1), as drop-in `target:`s:

* `ConcatTimestepEmbedderND` (encoders/modules.py:1000-1016): every scalar of x[b, d] -> sinusoidal embedding of `outdim`
  (util.py:207-231), concatenated to [b, d*outdim]. Used for fps_id / motion_bucket_id / cond_aug (infer_kubric.yaml:57-66,98-103).
* `SphericalEmbedder` (encoders/modules.py:247-287): (azimuth, elevation, radius) -> 13 trigonometric features -> Linear(13, dim).

Both run as one CUDA kernel each from libgcd_b200.so; like the rest of the package there is no CPU path. The properties the
reference's GeneralConditioner reads from AbstractEmbModel (is_trainable / ucg_rate / input_key, encoders/modules.py:40-81) exist.
"""
import torch
import torch.nn as nn

from . import ops


def _reference_base():
    """The reference GeneralConditioner asserts `isinstance(embedder, AbstractEmbModel)` (encoders/modules.py:93-96): when
    `sgm` imports, derive from its AbstractEmbModel so a YAML `target:` swap passes that gate; standalone, a plain nn.Module
    carrying the same three attributes (encoders/modules.py:40-81)."""
    try:
        from sgm.modules.encoders.modules import AbstractEmbModel as Ref   # noqa: WPS433
        return Ref
    except Exception:
        return nn.Module


_RefBase = _reference_base()


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
