"""H100-native temporal VAE decoder: drop-in for `sgm.modules.autoencoding.temporal_ae.VideoDecoder`
(temporal_ae.py:293-349 over diffusionmodules/model.py:604-748), time_mode "conv-only" (the default, :302).

`DiffusionEngine.decode_first_stage` gates on `isinstance(decoder, VideoDecoder)` (models/diffusion.py:242,620), so
`VideoDecoder` here is built as a real subclass of the reference class whenever `sgm` is importable (its heavy
__init__ is bypassed); standalone it is a plain nn.Module. State-dict keys equal the reference's
(`first_stage_model.decoder.*`, gcd_b200/spec.py).

Execution: channels-last, fp32 residual stream, 16-bit tensor-core operands, all compute in libgcd_b200.so kernels:
3x3 / (3,1,1) convs = wgmma implicit GEMM with fused bias/residual/alpha-blend epilogues, GroupNorm+SiLU streaming
kernels, the single-head d=512 mid attention as batched wgmma GEMMs (QK^T, PV) + a row-softmax kernel.
"""
import torch
import torch.nn as nn

from . import ops, spec
from .engine import Engine, EngineCache, need_option, reference_base, register_param_tree


class _VAEEngine(Engine):
    """What the VAE encoder and decoder share: channels-last fp32 residual stream, 16-bit tensor-core operands, the spatial
    ResnetBlock and the mid AttnBlock."""

    def __init__(self, cfg, plan, device):
        super().__init__(device)
        self.cfg, self.plan = cfg, plan

    def _pack_res(self, sd, p, cin, cout):
        self._norm(sd, p + ".n1", p + ".norm1")
        self._conv3(sd, p + ".c1", p + ".conv1")
        self._norm(sd, p + ".n2", p + ".norm2")
        self._conv3(sd, p + ".c2", p + ".conv2")
        if cin != cout:
            self._lin(sd, p + ".skip", p + ".nin_shortcut")

    def _pack_attn(self, sd, p):
        self._norm(sd, p + ".norm", p + ".norm")
        for n in ("q", "k", "v", "proj_out"):
            self._lin(sd, f"{p}.{n}", f"{p}.{n}")

    def _res2d(self, p, x, cin, cout, n, H, Wd, tag, out_geom, x_stats=None):
        """ResnetBlock.forward with temb=None (model.py:127-151). `out_geom`: (images, rows per image) of the GroupNorm that
        consumes the output, whose statistics conv2 accumulates. Returns (x_out fp32, those statistics or None)."""
        W, pool, AD = self.w, self.pool, self.AD
        HW, rows = H * Wd, n * H * Wd
        a = pool.get(f"a{cin}_{rows}", (rows, cin), AD)
        self._gn(x, n, HW, cin, p + ".n1", 1e-6, True, a, stats=x_stats)
        h1 = pool.get(f"h{cout}_{rows}", (rows, cout), AD)
        st, req = self._stats_req(n, cout, HW)
        ok = ops.conv2d_3x3(a.view(n, H, Wd, cin), W[p + ".c1.w"], ops.make_ep(h1, bias=W[p + ".c1.b"], gn_stats=req))
        a2 = pool.get(f"a{cout}_{rows}", (rows, cout), AD)
        self._gn(h1, n, HW, cout, p + ".n2", 1e-6, True, a2, stats=st if ok else None)
        xs = pool.get(f"{tag}_{cout}_{rows}", (rows, cout), torch.float32)
        if cin != cout:
            xa = pool.get(f"xa{cin}_{rows}", (rows, cin), AD)
            ops.cast_to_act(x, xa)
            ops.linear(xa, W[p + ".skip.w"], ops.make_ep(xs, bias=W[p + ".skip.b"]))
            res = xs
        else:
            res = x
        st, req = self._stats_req(out_geom[0], cout, out_geom[1])
        ok = ops.conv2d_3x3(a2.view(n, H, Wd, cout), W[p + ".c2.w"], ops.make_ep(xs, bias=W[p + ".c2.b"], res1=res, gn_stats=req))
        return xs, (st if ok else None)

    def _attn(self, p, x, C, n, S, x_stats=None):
        """AttnBlock (model.py:161-201): out = x + proj_out(softmax(q k^T / sqrt(C)) v), single head, per frame."""
        W, pool, AD = self.w, self.pool, self.AD
        rows = n * S
        a = pool.get(f"a{C}_{rows}", (rows, C), AD)
        self._gn(x, n, S, C, p + ".norm", 1e-6, False, a, stats=x_stats)
        q = pool.get("attn_q", (rows, C), AD)
        k = pool.get("attn_k", (rows, C), AD)
        ops.linear(a, W[p + ".q.w"], ops.make_ep(q, bias=W[p + ".q.b"]))
        ops.linear(a, W[p + ".k.w"], ops.make_ep(k, bias=W[p + ".k.b"]))
        vt = pool.get("attn_vt", (n, C, S), AD)                       # V^T per frame (K-major operand of P.V)
        for f in range(n):
            ops.linear(W[p + ".v.w"], a[f * S:(f + 1) * S], ops.make_ep(vt[f]))
        # chunk frames so the fp32 score matrix stays <= ~2.5 GB
        fc = max(1, min(n, int(2.5e9 // (S * S * 4))))
        o = pool.get("attn_o", (rows, C), AD)
        for f0 in range(0, n, fc):
            f1 = min(n, f0 + fc)
            sc = pool.get("attn_s", (fc * S, S), torch.float32)[: (f1 - f0) * S]
            pr = pool.get("attn_p", (fc * S, S), AD)[: (f1 - f0) * S]
            ops.bmm_nt(q[f0 * S:f1 * S].view(f1 - f0, S, C), k[f0 * S:f1 * S].view(f1 - f0, S, C), ops.make_ep(sc))
            ops.softmax_rows(sc, C ** -0.5, pr)
            # softmax rows sum to 1 => the v bias contributes exactly +b_v to every output row
            ops.bmm_nt(pr.view(f1 - f0, S, S), vt[f0:f1], ops.make_ep(o[f0 * S:f1 * S], bias=W[p + ".v.b"]))
        ops.linear(o, W[p + ".proj_out.w"], ops.make_ep(x, bias=W[p + ".proj_out.b"], res1=x))
        return x


class DecoderEngine(_VAEEngine):
    def __init__(self, cfg, state, device):
        super().__init__(cfg, spec.decoder_plan(cfg), device)
        self._pack(state)

    def _pack(self, sd):
        for kind, p, cin, cout in self.plan:
            if kind == "conv_in":
                self._conv3(sd, p, p, cin_pad=64)
            elif kind == "res":
                self._pack_res(sd, p, cin, cout)
                q = p + ".time_stack"
                self._norm(sd, q + ".n1", q + ".in_layers.0")
                self._convt(sd, q + ".c1", q + ".in_layers.2")
                self._norm(sd, q + ".n2", q + ".out_layers.0")
                self._convt(sd, q + ".c2", q + ".out_layers.3")
                self.alpha[p] = float(torch.sigmoid(self._f32(sd[p + ".mix_factor"])).item())
            elif kind == "attn":
                self._pack_attn(sd, p)
            elif kind == "up":
                self._conv3(sd, p, p + ".conv")
            elif kind == "out":
                self._norm(sd, "norm_out", "norm_out")
                self._conv3(sd, "conv_out", "conv_out")
                self.w["tmix.w"] = self._f32(sd["conv_out.time_mix_conv.weight"]).reshape(-1).contiguous()   # [co, ci, kt, 1, 1]
                self.w["tmix.b"] = self._f32(sd["conv_out.time_mix_conv.bias"]).contiguous()

    def _res(self, p, x, cin, cout, n, B, T, H, Wd, tag, x_stats=None):
        """temporal_ae.VideoResBlock.forward (temporal_ae.py:64-83) over ResnetBlock.forward (model.py:127-151).
        Returns (x_out, per-frame GroupNorm statistics of x_out or None)."""
        W, pool, AD = self.w, self.pool, self.AD
        HW, rows = H * Wd, n * H * Wd
        xs, st = self._res2d(p, x, cin, cout, n, H, Wd, tag, (B, T * HW), x_stats=x_stats)
        h1, a2 = pool.get(f"h{cout}_{rows}", (rows, cout), AD), pool.get(f"a{cout}_{rows}", (rows, cout), AD)
        q = p + ".time_stack"
        self._gn(xs, B, T * HW, cout, q + ".n1", 1e-5, True, a2, stats=st)
        st, req = self._stats_req(B, cout, T * HW)
        ok = ops.conv_t3(a2.view(B, T, HW, cout), W[q + ".c1.w"], ops.make_ep(h1, bias=W[q + ".c1.b"], gn_stats=req))
        self._gn(h1, B, T * HW, cout, q + ".n2", 1e-5, True, a2, stats=st if ok else None)
        # x = alpha * (x_s + conv) + (1 - alpha) * x_s = x_s + alpha * conv     (temporal_ae.py:79-80)
        st, req = self._stats_req(n, cout, HW)
        ok = ops.conv_t3(a2.view(B, T, HW, cout), W[q + ".c2.w"],
                         ops.make_ep(xs, bias=W[q + ".c2.b"], a_acc=self.alpha[p], res1=xs, gn_stats=req))
        return xs, (st if ok else None)

    def forward_cl(self, z_cl, n, H, Wd, T, out_nchw):
        """z_cl: act channels-last [n, H, W, 64]; writes float32 NCHW [n, out_ch, 8H, 8W] into out_nchw."""
        W, pool, AD = self.w, self.pool, self.AD
        assert n % T == 0
        B = n // T
        self.arena.reset(n)
        h, hH, hW, hC, hst = None, H, Wd, None, None
        for i, (kind, p, cin, cout) in enumerate(self.plan):
            rows = n * hH * hW
            if kind == "conv_in":
                h = pool.get(f"s0_{cout}_{rows}", (rows, cout), torch.float32)
                st, req = self._stats_req(n, cout, hH * hW)
                ok = ops.conv2d_3x3(z_cl, W[p + ".w"], ops.make_ep(h, bias=W[p + ".b"], gn_stats=req))
                hC, hst = cout, (st if ok else None)
            elif kind == "res":
                h, hst = self._res(p, h, cin, cout, n, B, T, hH, hW, f"s{1 + i % 2}", x_stats=hst)
                hC = cout
            elif kind == "attn":
                h = self._attn(p, h, cin, n, hH * hW, x_stats=hst)
                hst = None
            elif kind == "up":
                xu = pool.get(f"up{cin}_{rows * 4}", (rows * 4, cin), AD)
                ops.upsample2x_to_act(h, n, hH, hW, cin, xu)
                # the lower level's workspaces are dead from here on: free them, so that the decoder's peak is its largest
                # level alone (14 frames at 576x1024 px would otherwise hold every level's buffers at once, ~55 GB)
                pool.release_rows(rows)
                hH, hW = 2 * hH, 2 * hW
                h = pool.get(f"s0_{cout}_{rows * 4}", (rows * 4, cout), torch.float32)
                st, req = self._stats_req(n, cout, hH * hW)
                ok = ops.conv2d_3x3(xu.view(n, hH, hW, cin), W[p + ".w"], ops.make_ep(h, bias=W[p + ".b"], gn_stats=req))
                hst = st if ok else None
                pool.release(f"up{cin}_{rows * 4}")            # the upsampled input is dead once the conv has read it
                del xu
            elif kind == "out":
                a = pool.get(f"a{cin}_{rows}", (rows, cin), AD)
                self._gn(h, n, hH * hW, cin, "norm_out", 1e-6, True, a, stats=hst)
                o16 = pool.get(f"out16_{rows}", (rows, 16), torch.float32)
                ops.conv2d_3x3(a.view(n, hH, hW, cin), W["conv_out.w"], ops.make_ep(o16[:, :cout], bias=W["conv_out.b"]))
                assert cout == 3, "AE3DConv tail kernel is written for 3 output channels"
                ops.vae_time_mix(o16, 16, B, T, hH * hW, W["tmix.w"], W["tmix.b"], out_nchw)
        return out_nchw


class EncoderEngine(_VAEEngine):
    """VAE Encoder of the conditioning frames (diffusionmodules/model.py:487-601; SURVEY.md §8(f) rank 1): the same
    channels-last fp32-residual design and the same kernels as the decoder, plus the stride-2 (0,1,0,1)-padded Downsample conv.

    `post=(Wq [co, 2z], bq [co], scale)` folds a following 1x1 conv and scale into conv_out — exact algebra:
    scale * (Wq (W_out * h + b_out) + bq) = (scale Wq W_out) * h + scale (Wq b_out + bq). AutoencoderKLModeOnly
    (autoencoder.py:493-513,627-640) is quant_conv followed by "take the mean half", i.e. post = (Wq[:z], bq[:z], scale_factor).
    """

    def __init__(self, cfg, state, device, post=None):
        super().__init__(cfg, spec.encoder_plan(cfg), device)
        self._pack(state, post)

    def _pack(self, sd, post):
        for kind, p, cin, cout in self.plan:
            if kind == "conv_in":
                self._conv3(sd, p, p, cin_pad=64)
            elif kind == "res":
                self._pack_res(sd, p, cin, cout)
            elif kind == "attn":
                self._pack_attn(sd, p)
            elif kind == "down":
                self._conv3(sd, p, p + ".conv")
            elif kind == "out":
                self._norm(sd, "norm_out", "norm_out")
                w, b = self._f32(sd["conv_out.weight"]), self._f32(sd["conv_out.bias"])
                if post is not None:
                    wq, bq, scale = post
                    wq, bq = self._f32(wq).reshape(wq.shape[0], -1), self._f32(bq)
                    w = float(scale) * torch.einsum("oc,cikl->oikl", wq, w)
                    b = float(scale) * (wq @ b + bq)
                self.out_ch = w.shape[0]
                assert self.out_ch <= 16
                self._conv3(sd, "conv_out", (w, b))

    def forward_cl(self, x_cl, n, H, Wd, out_nchw):
        """x_cl: act channels-last [n, H, W, 64] (image channels zero-padded); writes float32 NCHW [n, out_ch, H/8, W/8]."""
        W, pool, AD = self.w, self.pool, self.AD
        self.arena.reset(n)
        h, hH, hW, hst = None, H, Wd, None
        for i, (kind, p, cin, cout) in enumerate(self.plan):
            rows = n * hH * hW
            if kind == "conv_in":
                h = pool.get(f"s0_{cout}_{rows}", (rows, cout), torch.float32)
                st, req = self._stats_req(n, cout, hH * hW)
                ok = ops.conv2d_3x3(x_cl, W[p + ".w"], ops.make_ep(h, bias=W[p + ".b"], gn_stats=req))
                hst = st if ok else None
            elif kind == "res":
                h, hst = self._res2d(p, h, cin, cout, n, hH, hW, f"s{1 + i % 2}", (n, hH * hW), x_stats=hst)
            elif kind == "attn":
                h = self._attn(p, h, cin, n, hH * hW, x_stats=hst)
                hst = None
            elif kind == "down":
                assert hH % 2 == 0 and hW % 2 == 0, "Downsample expects even sizes (the reference pads (0,1,0,1) and floors)"
                xa = pool.get(f"dn{cin}_{rows}", (rows, cin), AD)
                ops.cast_to_act(h, xa)
                h = pool.get(f"s0_{cout}_{rows // 4}", (rows // 4, cout), torch.float32)
                st, req = self._stats_req(n, cout, (hH // 2) * (hW // 2))
                ok = ops.conv2d_3x3_down_pad01(xa.view(n, hH, hW, cin), W[p + ".w"], ops.make_ep(h, bias=W[p + ".b"], gn_stats=req))
                hH, hW = hH // 2, hW // 2
                hst = st if ok else None
            elif kind == "out":
                a = pool.get(f"a{cin}_{rows}", (rows, cin), AD)
                self._gn(h, n, hH * hW, cin, "norm_out", 1e-6, True, a, stats=hst)
                o16 = pool.get(f"out16_{rows}", (rows, 16), torch.float32)
                ops.conv2d_3x3(a.view(n, hH, hW, cin), W["conv_out.w"], ops.make_ep(o16[:, :self.out_ch], bias=W["conv_out.b"]))
                ops.nhwc_to_nchw(o16, 16, n, self.out_ch, hH * hW, out_nchw)
        return out_nchw


class Encoder(nn.Module):
    """Drop-in `target:` for sgm.modules.diffusionmodules.model.Encoder (ctor kwargs: infer_kubric.yaml:83-94); state-dict
    keys equal the reference's (`...encoder.encoder.*`). forward(x [n, 3, H, W]) -> moments [n, 2*z_channels, H/8, W/8].
    `encode_mode` is the fused AutoencoderKLModeOnly.encode + VideoPredictionEmbedderWithEncoder scale (modules.py:1100-1106)."""

    def __init__(self, *, ch, out_ch=3, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions=(), dropout=0.0,
                 resamp_with_conv=True, in_channels, resolution=256, z_channels, double_z=True, use_linear_attn=False,
                 attn_type="vanilla", **ignore_kwargs):
        super().__init__()
        need = need_option("Encoder")
        need(len(attn_resolutions) == 0 and attn_type in ("vanilla", "vanilla-xformers") and not use_linear_attn, "attention")
        need(resamp_with_conv and dropout == 0.0, "resamp_with_conv / dropout")
        need(ch % 64 == 0 and in_channels <= 64 and (2 if double_z else 1) * z_channels <= 16, "channel counts")
        self.cfg = dict(ch=ch, ch_mult=list(ch_mult), num_res_blocks=num_res_blocks, z_channels=z_channels,
                        in_channels=in_channels, double_z=double_z)
        register_param_tree(self, spec.encoder_param_shapes(self.cfg))
        self._engines = EngineCache(slots=2)

    def invalidate(self):
        self._engines.clear()

    def engine(self, device, post=None, post_key=None):
        """One packed engine per `post` fold (plain forward / encode_mode), at most two kept; a weight change drops them all."""
        return self._engines.get(self, device, lambda: EncoderEngine(self.cfg, self.state_dict(), device, post=post), post_key)

    def _run(self, x, eng):
        if not x.is_cuda:
            raise RuntimeError("gcd_b200.Encoder runs on CUDA (sm_90a) only; there is no CPU path")
        n, c, H, W = x.shape
        ndown = len(self.cfg["ch_mult"]) - 1
        if c != self.cfg["in_channels"] or H % (1 << ndown) or W % (1 << ndown) or ((H >> ndown) * (W >> ndown)) % 8:
            raise ValueError(f"Encoder input must be [n, {self.cfg['in_channels']}, H, W] with H, W multiples of {1 << ndown} "
                             f"and (H/{1 << ndown})*(W/{1 << ndown}) a multiple of 8 (16-byte rows of the mid-attention scores)")
        x_cl = eng.pool.get("x_cl", (n, H, W, 64), eng.AD)
        ops.nchw_to_act_nhwc(x.to(torch.float32).contiguous(), n, c, H * W, 64, x_cl)
        out = torch.empty(n, eng.out_ch, H >> ndown, W >> ndown, device=x.device, dtype=torch.float32)
        eng.forward_cl(x_cl, n, H, W, out)
        return out.to(x.dtype)

    @torch.no_grad()
    def forward(self, x):
        return self._run(x, self.engine(x.device))

    @torch.no_grad()
    def encode_mode(self, x, quant_weight, quant_bias, scale_factor=1.0):
        """scale_factor * mode(DiagonalGaussian(quant_conv(encoder(x)))) = the first z_channels of quant_conv's output."""
        z = self.cfg["z_channels"]
        post = (quant_weight[:z], quant_bias[:z], scale_factor)
        # keyed on the CONTENT of the (tiny: 2z x 2z) quant_conv so a freshly materialised tensor with the same values hits
        pk = (tuple(quant_weight.detach().double().flatten().tolist()), tuple(quant_bias.detach().double().flatten().tolist()),
              float(scale_factor))
        return self._run(x, self.engine(x.device, post=post, post_key=pk))


class VideoDecoder(reference_base("sgm.modules.autoencoding.temporal_ae", "VideoDecoder")):
    """Drop-in `target:` for sgm.modules.autoencoding.temporal_ae.VideoDecoder (ctor kwargs: infer_kubric.yaml:152-164)."""

    def __init__(self, *args, ch, out_ch, ch_mult=(1, 2, 4, 8), num_res_blocks, attn_resolutions=(), dropout=0.0,
                 resamp_with_conv=True, in_channels=3, resolution=256, z_channels, give_pre_end=False, tanh_out=False,
                 use_linear_attn=False, attn_type="vanilla", video_kernel_size=3, alpha=0.0, merge_strategy="learned",
                 time_mode="conv-only", **ignorekwargs):
        nn.Module.__init__(self)   # bypass the reference constructor (it would build the eager torch layers)
        need = need_option("VideoDecoder")
        need(time_mode == "conv-only" and merge_strategy == "learned", "time_mode/merge_strategy")
        need(len(attn_resolutions) == 0 and attn_type in ("vanilla", "vanilla-xformers") and not use_linear_attn, "attention")
        need(resamp_with_conv and not give_pre_end and not tanh_out and dropout == 0.0, "decoder flags")
        need(list(video_kernel_size) == [3, 1, 1] if not isinstance(video_kernel_size, int) else False, "video_kernel_size")
        need(out_ch == 3 and ch % 64 == 0, "out_ch must be 3, ch a multiple of 64")
        self.cfg = dict(ch=ch, out_ch=out_ch, ch_mult=list(ch_mult), num_res_blocks=num_res_blocks, z_channels=z_channels)
        self.time_mode, self.video_kernel_size, self.alpha, self.merge_strategy = time_mode, video_kernel_size, alpha, merge_strategy
        register_param_tree(self, spec.decoder_param_shapes(self.cfg))
        self._engines = EngineCache()

    def get_last_layer(self, skip_time_mix=False, **kwargs):
        return self.conv_out.time_mix_conv.weight if not skip_time_mix else self.conv_out.weight

    def invalidate(self):
        self._engines.clear()

    def engine(self, device):
        return self._engines.get(self, device, lambda: DecoderEngine(self.cfg, self.state_dict(), device))

    @torch.no_grad()
    def forward(self, z, timesteps=None, skip_video=False, **kwargs):
        if not z.is_cuda:
            raise RuntimeError("gcd_b200.VideoDecoder runs on CUDA (sm_90a) only; there is no CPU path")
        if skip_video or timesteps is None:
            raise NotImplementedError("VideoDecoder needs timesteps=<frames per clip> and skip_video=False")
        n, c, H, W = z.shape
        eng = self.engine(z.device)
        z_cl = eng.pool.get("z_cl", (n, H, W, 64), eng.AD)
        ops.nchw_to_act_nhwc(z.to(torch.float32).contiguous(), n, c, H * W, 64, z_cl)
        nup = len(self.cfg["ch_mult"]) - 1
        out = torch.empty(n, self.cfg["out_ch"], H << nup, W << nup, device=z.device, dtype=torch.float32)
        eng.forward_cl(z_cl, n, H, W, int(timesteps), out)
        return out.to(z.dtype)
