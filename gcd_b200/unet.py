"""H100-native VideoUNet: drop-in for `sgm.modules.diffusionmodules.video_model.VideoUNet` (video_model.py:84-540).

* `VideoUNet` is an nn.Module with the reference constructor kwargs, the reference `state_dict` keys/shapes
  (gcd_b200/spec.py) and the reference `forward` signature, so `instantiate_from_config` + `init_from_ckpt`
  (models/diffusion.py:76-79,191-219) work unchanged by switching the YAML `target:`.
* `UNetEngine` is the execution plan underneath: weights repacked once to kernel-native fp16 layouts, activations kept
  channels-last `[frames, H*W, C]` (residual stream fp32, tensor-core operands 16-bit), every block executed by the
  hand-written sm_90a kernels of libgcd_b200.so through gcd_b200.ops. There is no PyTorch compute fallback.

Exact algebraic shortcuts taken (SURVEY.md §8(a) facts 1-5, all parity-tested against the oracle):
  - cross-attention context length is 1 in GCD => attn2(x, ctx) == to_out(to_v(ctx)): a per-frame (spatial) / per-clip
    (temporal, context[::T]) vector added in the self-attention out-projection epilogue;
  - `time_pos_embed(timestep_embedding(arange(T)))` is input independent => computed once at pack time;
  - all 50 `emb_layers` Linear(SiLU(emb)) run as one GEMM per forward;
  - image_only_indicator is all zeros => AlphaBlender alpha = sigmoid(mix_factor) (scalar per blender).
"""
import os

import torch
import torch.nn as nn

from . import ops, spec
from .engine import Engine, EngineCache, need_option, register_param_tree


def _geglu_interleave(w, b):
    """Rows [0,H) value / [H,2H) gate (attention.py:93 chunk) -> blocks of 16 value rows followed by 16 gate rows."""
    H = w.shape[0] // 2
    idx = torch.arange(2 * H, device=w.device).view(2, H // 16, 16).permute(1, 0, 2).reshape(-1)
    return w[idx].contiguous(), b[idx].contiguous()


# ----------------------------------------------------------------------------------------------------------------------
class UNetEngine(Engine):
    def __init__(self, cfg, state, device):
        """state: mapping reference-key -> float32 tensor (any device)."""
        super().__init__(device)
        self.cfg = cfg
        self.plan = spec.unet_plan(cfg)
        self._pe_cache = {}
        self.debug = None          # set to a list to record every layer's output (tools/bisect_batch.py)
        self.use_graphs = os.environ.get("GCD_NO_GRAPH", "0") != "1"
        self._graphs = {}
        self._pack(state)

    # ------------------------------------------------------------------------------------------------ weight packing
    def _pack(self, sd):
        g = lambda k: self._f32(sd[k])

        def attn(p):
            qkv = [g(p + ".attn1.to_q.weight"), g(p + ".attn1.to_k.weight"), g(p + ".attn1.to_v.weight")]
            self._lin(sd, p + ".qkv", (torch.cat(qkv, 0), None))     # the fp32 concatenation is freed right after packing
            self._lin(sd, p + ".attn1.out", p + ".attn1.to_out.0")
            self._lin(sd, p + ".attn2.v", p + ".attn2.to_v")
            self._lin(sd, p + ".attn2.out", p + ".attn2.to_out.0")

        def geglu(name, key):
            self._lin(sd, name, _geglu_interleave(g(key + ".weight"), g(key + ".bias")))

        for k in ("time_embed.0", "time_embed.2", "label_emb.0.0", "label_emb.0.2"):
            self._lin(sd, k, k)
        if self.cfg["aux_emb_dim"] > 0:
            self._lin(sd, "aux_label_emb.0", "aux_label_emb.0")
            self._lin(sd, "aux_label_emb.2", "aux_label_emb.2")
        inp, mid, out = self.plan
        emb_w, emb_b, self.emb_off, off = [], [], {}, 0
        for layers in inp + [mid] + out:
            for kind, p, cin, cout in layers:
                if kind == "conv_in":
                    self._conv3(sd, p, p, cin_pad=64)
                elif kind == "down":
                    self._conv3(sd, p, p + ".op")
                elif kind == "up":
                    self._conv3(sd, p, p + ".conv")
                elif kind == "vrb":
                    self._norm(sd, p + ".n1", p + ".in_layers.0")
                    self._conv3(sd, p + ".c1", p + ".in_layers.2")
                    self._norm(sd, p + ".n2", p + ".out_layers.0")
                    self._conv3(sd, p + ".c2", p + ".out_layers.3")
                    if cin != cout:
                        self._lin(sd, p + ".skip", p + ".skip_connection")
                    q = p + ".time_stack"
                    self._norm(sd, q + ".n1", q + ".in_layers.0")
                    self._convt(sd, q + ".c1", q + ".in_layers.2")
                    self._norm(sd, q + ".n2", q + ".out_layers.0")
                    self._convt(sd, q + ".c2", q + ".out_layers.3")
                    for e in (p, q):
                        emb_w.append(g(e + ".emb_layers.1.weight"))
                        emb_b.append(g(e + ".emb_layers.1.bias"))
                        self.emb_off[e] = off
                        off += cout
                    self.alpha[p] = float(torch.sigmoid(g(p + ".time_mixer.mix_factor")).item())
                elif kind == "svt":
                    self._norm(sd, p + ".norm", p + ".norm")
                    self._lin(sd, p + ".proj_in", p + ".proj_in")
                    self._lin(sd, p + ".proj_out", p + ".proj_out")
                    assert self.cfg["transformer_depth"] == 1, "transformer_depth != 1 is not used by GCD"
                    s, t = p + ".transformer_blocks.0", p + ".time_stack.0"
                    for blk in (s, t):
                        attn(blk)
                        for n in ("norm1", "norm3") + (("norm_in",) if blk == t else ()):
                            self._norm(sd, blk + "." + n, blk + "." + n)
                        geglu(blk + ".ff.0", blk + ".ff.net.0.proj")
                        self._lin(sd, blk + ".ff.2", blk + ".ff.net.2")
                    geglu(t + ".ff_in.0", t + ".ff_in.net.0.proj")
                    self._lin(sd, t + ".ff_in.2", t + ".ff_in.net.2")
                    self._lin(sd, p + ".tpe.0", p + ".time_pos_embed.0")
                    self._lin(sd, p + ".tpe.2", p + ".time_pos_embed.2")
                    self.alpha[p] = float(torch.sigmoid(g(p + ".time_mixer.mix_factor")).item())
        self._lin(sd, "emb_all", (torch.cat(emb_w, 0), torch.cat(emb_b, 0)))
        self.emb_total = off
        self._norm(sd, "out.0", "out.0")
        self._conv3(sd, "out.2", "out.2")

    # ------------------------------------------------------------------------------------------------ small helpers
    def _mlp_small(self, x_act, k0, k2, out_f32, accumulate):
        """Linear -> SiLU -> Linear on a handful of rows (time_embed / label_emb / time_pos_embed)."""
        W = self.w
        hid = self.pool.get("mlp_hid", (x_act.shape[0], W[k0 + ".w"].shape[0]), self.AD)
        ops.linear(x_act, W[k0 + ".w"], ops.make_ep(hid, bias=W[k0 + ".b"], act=1))
        ops.linear(hid, W[k2 + ".w"], ops.make_ep(out_f32, bias=W[k2 + ".b"], res1=out_f32 if accumulate else None))

    def _pos_embed(self, p, T, C):
        """time_pos_embed(timestep_embedding(arange(T), C)) (video_attention.py:266-276): [T, C] float32, cached."""
        key = (p, T)
        if key not in self._pe_cache:
            t = torch.arange(T, device=self.device, dtype=torch.float32)
            te = torch.empty(T, C, device=self.device, dtype=self.AD)
            ops.timestep_embedding(t, C, out_act=te)
            pe = torch.empty(T, C, device=self.device, dtype=torch.float32)
            self._mlp_small(te, p + ".tpe.0", p + ".tpe.2", pe, False)
            self._pe_cache[key] = pe
        return self._pe_cache[key]

    def _pos_embed_frames(self, p, T, C, n):
        """The [T, C] time position embedding laid out per frame of the batch ([n, C], frame f -> t = f % T): a rowvec operand."""
        key = (p, T, n)
        if key not in self._pe_cache:
            self._pe_cache[key] = self._pos_embed(p, T, C).repeat(n // T, 1).contiguous()
        return self._pe_cache[key]

    def cross_attn_vectors(self, context, T, static=False):
        """len-1 cross attention == to_out(to_v(ctx)) (+bias): per frame for the spatial blocks, per clip
        (context[::T], video_attention.py:249-253) for the temporal blocks. Step-invariant: the fused sampler computes
        it once per sample and passes it to every step; a plain forward() recomputes it (no pointer-keyed caching —
        a recycled allocation with new contents must never hit a stale entry). `static`: write into pool buffers (fixed
        addresses across samples, so a captured CUDA graph of the forward can be replayed for the next sample)."""
        if context.dim() != 3 or context.shape[1] != 1:
            raise NotImplementedError(
                f"gcd_b200.VideoUNet supports the GCD conditioning layout context=[BT,1,D] only, got {tuple(context.shape)}")
        ctx = context[:, 0, :].to(self.device, torch.float32).to(self.AD).contiguous()
        ctx_t = ctx[::T].contiguous()
        vecs = {}
        inp, mid, out = self.plan
        for layers in inp + [mid] + out:
            for kind, p, cin, cout in layers:
                if kind != "svt":
                    continue
                for blk, c in ((p + ".transformer_blocks.0", ctx), (p + ".time_stack.0", ctx_t)):
                    if static:
                        v = self.pool.get("ca_v", (c.shape[0], cout), self.AD)
                        o = self.pool.get("ca:" + blk, (c.shape[0], cout), torch.float32)
                    else:
                        v = torch.empty(c.shape[0], cout, device=self.device, dtype=self.AD)
                        o = torch.empty(c.shape[0], cout, device=self.device, dtype=torch.float32)
                    ops.linear(c, self.w[blk + ".attn2.v.w"], ops.make_ep(v))
                    ops.linear(v, self.w[blk + ".attn2.out.w"], ops.make_ep(o, bias=self.w[blk + ".attn2.out.b"]))
                    vecs[blk] = o
        return vecs

    # ------------------------------------------------------------------------------------------------ blocks
    def _vrb(self, p, x, cin, cout, n, B, T, H, Wd, emb_all, out=None, x_stats=None):
        """VideoResBlock.forward (video_model.py:62-81) over ResBlock._forward (openaimodel.py:331-357).
        x: float32 [n*H*W, cin]; returns (float32 [n*H*W, cout], per-frame GroupNorm statistics of it or None).
        Every conv accumulates the statistics of the GroupNorm that follows it in its epilogue (gcd_epilogue.gn_stats)."""
        W, pool, AD = self.w, self.pool, self.AD
        HW = H * Wd
        rows = n * HW
        a = pool.get(f"act_a{cin}", (rows, cin), AD)
        self._gn(x, n, HW, cin, p + ".n1", 1e-5, True, a, stats=x_stats)
        h1 = pool.get(f"act_h{cout}", (rows, cout), AD)
        eo = self.emb_off[p]
        st, req = self._stats_req(n, cout, HW)
        ok = ops.conv2d_3x3(a.view(n, H, Wd, cin), W[p + ".c1.w"],
                            ops.make_ep(h1, bias=W[p + ".c1.b"], rowvec=emb_all[:, eo:eo + cout], rows_per_vec=HW, gn_stats=req))
        a2 = pool.get(f"act_a{cout}", (rows, cout), AD)
        self._gn(h1, n, HW, cout, p + ".n2", 1e-5, True, a2, stats=st if ok else None)
        xs = out if out is not None else pool.get(f"vrb_xs{cout}", (rows, cout), torch.float32)
        if cin != cout:
            if x.dtype == AD:                        # 16-bit skip concat (forward_cl): already the skip conv's operand
                xa = x
            else:
                xa = pool.get(f"act_x{cin}", (rows, cin), AD)
                ops.cast_to_act(x, xa)
            ops.linear(xa, W[p + ".skip.w"], ops.make_ep(xs, bias=W[p + ".skip.b"]))
            res = xs
        else:
            assert x.dtype == torch.float32, "identity skip needs the fp32 residual stream"
            res = x
        st, req = self._stats_req(B, cout, T * HW)
        ok = ops.conv2d_3x3(a2.view(n, H, Wd, cout), W[p + ".c2.w"],
                            ops.make_ep(xs, bias=W[p + ".c2.b"], res1=res, gn_stats=req))
        # ---- temporal ResBlock (time_stack) + AlphaBlender; its GroupNorms span (C/32, T, H, W) per clip
        q = p + ".time_stack"
        self._gn(xs, B, T * HW, cout, q + ".n1", 1e-5, True, a2, stats=st if ok else None)
        eo = self.emb_off[q]
        st, req = self._stats_req(B, cout, T * HW)
        ok = ops.conv_t3(a2.view(B, T, HW, cout), W[q + ".c1.w"],
                         ops.make_ep(h1, bias=W[q + ".c1.b"], rowvec=emb_all[:, eo:eo + cout], rows_per_vec=HW, gn_stats=req))
        self._gn(h1, B, T * HW, cout, q + ".n2", 1e-5, True, a2, stats=st if ok else None)
        al = self.alpha[p]
        # x = alpha * x_spatial + (1 - alpha) * (x_spatial + conv)  =  x_spatial + (1 - alpha) * conv
        st, req = self._stats_req(n, cout, HW)
        ok = ops.conv_t3(a2.view(B, T, HW, cout), W[q + ".c2.w"],
                         ops.make_ep(xs, bias=W[q + ".c2.b"], a_acc=1.0 - al, res1=xs, a_res1=1.0, gn_stats=req))
        return xs, (st if ok else None)

    def _ff(self, blk, name, a, rows, C, ep2):
        W = self.w
        hid = self.pool.get(f"ffh{C}", (rows, 4 * C), self.AD)
        ops.linear(a, W[f"{blk}.{name}.0.w"], ops.make_ep(hid, bias=W[f"{blk}.{name}.0.b"], geglu=True))
        ops.linear(hid, W[f"{blk}.{name}.2.w"], ep2)

    def _svt(self, p, xin, C, n, B, T, S, ca, x_stats=None):
        """SpatialVideoTransformer.forward (video_attention.py:230-301); xin float32 [n*S, C], updated in place.
        Returns (xin, per-frame GroupNorm statistics of the result or None)."""
        W, pool, AD = self.w, self.pool, self.AD
        rows = n * S
        heads = C // 64
        a = pool.get(f"act_a{C}", (rows, C), AD)
        self._gn(xin, n, S, C, p + ".norm", 1e-6, False, a, stats=x_stats)
        x = pool.get(f"svt_x{C}", (rows, C), torch.float32)
        ops.linear(a, W[p + ".proj_in.w"], ops.make_ep(x, bias=W[p + ".proj_in.b"]))
        # ---- spatial BasicTransformerBlock (attention.py:551-572)
        s = p + ".transformer_blocks.0"
        ops.layernorm(x, W[s + ".norm1.g"], W[s + ".norm1.b"], a)
        qkv = pool.get(f"qkv{C}", (rows, 3 * C), AD)
        ops.linear(a, W[s + ".qkv.w"], ops.make_ep(qkv))
        o = pool.get(f"act_h{C}", (rows, C), AD)
        ops.attention_spatial(qkv, n, S, heads, o)
        ops.linear(o, W[s + ".attn1.out.w"], ops.make_ep(x, bias=W[s + ".attn1.out.b"], res1=x, rowvec=ca[s], rows_per_vec=S))
        ops.layernorm(x, W[s + ".norm3.g"], W[s + ".norm3.b"], a)
        self._ff(s, "ff", a, rows, C, ops.make_ep(x, bias=W[s + ".ff.2.b"], res1=x))
        # ---- temporal VideoTransformerBlock (video_attention.py:109-140), tokens stay in (b t) s c order
        t = p + ".time_stack.0"
        pe = self._pos_embed(p, T, C)
        xm = pool.get(f"svt_xm{C}", (rows, C), torch.float32)
        # x_mix = x + time_pos_embed[t] is never materialised: norm_in adds the embedding on the fly, and the residual of ff_in
        # (x_mix + ff_in(norm_in(x_mix)), video_attention.py:118-121) is taken from x with the embedding as the per-frame vector of
        # the GEMM epilogue (folded into its bias slice) — saves the 4 B/element write-back of the sum
        ops.layernorm(x, W[t + ".norm_in.g"], W[t + ".norm_in.b"], a, add=pe, add_rows_per=S, add_mod=T)
        self._ff(t, "ff_in", a, rows, C, ops.make_ep(xm, bias=W[t + ".ff_in.2.b"], res1=x, rowvec=self._pos_embed_frames(p, T, C, n),
                                                     rows_per_vec=S))
        ops.layernorm(xm, W[t + ".norm1.g"], W[t + ".norm1.b"], a)
        ops.linear(a, W[t + ".qkv.w"], ops.make_ep(qkv))
        ops.attention_temporal(qkv, B, T, S, heads, o)
        ops.linear(o, W[t + ".attn1.out.w"],
                   ops.make_ep(xm, bias=W[t + ".attn1.out.b"], res1=xm, rowvec=ca[t], rows_per_vec=T * S))
        ops.layernorm(xm, W[t + ".norm3.g"], W[t + ".norm3.b"], a)
        al = self.alpha[p]
        # AlphaBlender (util.py:358-369): alpha * x + (1 - alpha) * (x_mix + ff(x_mix)) -> act operand of proj_out
        blended = pool.get(f"act_b{C}", (rows, C), AD)
        self._ff(t, "ff", a, rows, C, ops.make_ep(blended, bias=W[t + ".ff.2.b"], a_acc=1.0 - al, res1=xm, a_res1=1.0 - al,
                                                  res2=x, a_res2=al))
        st, req = self._stats_req(n, C, S)
        ok = ops.linear(blended, W[p + ".proj_out.w"], ops.make_ep(xin, bias=W[p + ".proj_out.b"], res1=xin, gn_stats=req))
        return xin, (st if ok else None)

    # ------------------------------------------------------------------------------------------------ forward
    def embed(self, timesteps, y):
        """video_model.py:483-497 -> all emb_layers outputs [n, emb_total] float32."""
        cfg, W, pool, AD = self.cfg, self.w, self.pool, self.AD
        n = timesteps.shape[0]
        mc = cfg["model_channels"]
        te = pool.get("t_emb", (n, mc), AD)
        ops.timestep_embedding(timesteps.to(torch.float32).contiguous(), mc, out_act=te)
        emb = pool.get("emb", (n, 4 * mc), torch.float32)
        self._mlp_small(te, "time_embed.0", "time_embed.2", emb, False)
        adm = cfg["adm_in_channels"]
        ya = y.to(self.device, torch.float32).to(AD)
        self._mlp_small(ya[:, :adm].contiguous(), "label_emb.0.0", "label_emb.0.2", emb, True)
        if cfg["aux_emb_dim"] > 0:
            assert y.shape[-1] == adm + cfg["aux_emb_dim"]
            self._mlp_small(ya[:, adm:].contiguous(), "aux_label_emb.0", "aux_label_emb.2", emb, True)
        es = pool.get("emb_silu", (n, 4 * mc), AD)
        ops.silu_f32_to_act(emb, es)
        emb_all = pool.get("emb_all", (n, self.emb_total), torch.float32)
        ops.linear(es, W["emb_all.w"], ops.make_ep(emb_all, bias=W["emb_all.b"]))
        return emb_all

    def forward_graphed(self, x_cl, n, H, Wd, timesteps, context, y, T, ca):
        """forward_cl replayed from a CUDA graph (SURVEY.md §7 step 7): ~620 kernel launches per CFG forward, each with six host
        `cuTensorMapEncodeTiled` calls and ctypes marshalling, become one `cudaGraphLaunch`. The tensor maps are
        __grid_constant__ kernel parameters, i.e. baked into the graph's kernel nodes, so every input must keep its ADDRESS
        between replays: the fused sampler passes pool buffers (x_cl, t_in, ctx / y copies, static cross-attention vectors).
        Keyed on shapes + those addresses; the first call for a key runs eagerly once (allocates workspaces, configures the
        kernels), captures, then replays. Disabled under ops.profile (per-launch events) and with GCD_NO_GRAPH=1."""
        if not self.use_graphs or ops._PROF is not None or self.debug is not None:
            return self.forward_cl(x_cl, n, H, Wd, timesteps, context, y, T, ca=ca)
        key = (n, H, Wd, T, x_cl.data_ptr(), timesteps.data_ptr(), context.data_ptr(), y.data_ptr(),
               tuple(v.data_ptr() for v in ca.values()))
        ent = self._graphs.get(key)
        if ent is None:
            self.forward_cl(x_cl, n, H, Wd, timesteps, context, y, T, ca=ca)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            l0 = ops.launch_count()
            with torch.cuda.graph(graph):
                res = self.forward_cl(x_cl, n, H, Wd, timesteps, context, y, T, ca=ca)
            if len(self._graphs) >= 4:
                self._graphs.pop(next(iter(self._graphs)))
            ent = self._graphs[key] = (graph, res, ops.launch_count() - l0)
        ent[0].replay()
        ops.count_replayed_launches(ent[2])
        return ent[1]

    def forward_cl(self, x_cl, n, H, Wd, timesteps, context, y, T, ca=None):
        """x_cl: act channels-last [n, H, W, 64] (first in_channels used). Returns float32 [n*H*W, 16]-strided buffer
        whose first out_channels columns hold the result (channels-last)."""
        cfg, W, pool, AD = self.cfg, self.w, self.pool, self.AD
        assert n % T == 0
        B = n // T
        self.arena.reset(n)
        emb_all = self.embed(timesteps, y)
        if ca is None:
            ca = self.cross_attn_vectors(context, T)
        inp, mid, out = self.plan
        hs = []
        h, hH, hW, hC = None, H, Wd, None

        def run(layers, h, hH, hW, hC, bi, tag, hst):
            """hst: per-frame GroupNorm statistics of h accumulated by its producer (or None)."""
            for kind, p, cin, cout in layers:
                rows = n * hH * hW
                if kind == "conv_in":
                    o = pool.get(f"{tag}{bi}", (rows, cout), torch.float32)
                    st, req = self._stats_req(n, cout, hH * hW)
                    ok = ops.conv2d_3x3(x_cl, W[p + ".w"], ops.make_ep(o, bias=W[p + ".b"], gn_stats=req))
                    h, hC, hst = o, cout, (st if ok else None)
                elif kind == "vrb":
                    o = pool.get(f"{tag}{bi}", (rows, cout), torch.float32)
                    h, hst = self._vrb(p, h, cin, cout, n, B, T, hH, hW, emb_all, out=o, x_stats=hst)
                    hC = cout
                elif kind == "svt":
                    h, hst = self._svt(p, h, cout, n, B, T, hH * hW, ca, x_stats=hst)
                elif kind == "down":
                    xa = pool.get(f"act_x{cin}", (rows, cin), AD)
                    ops.cast_to_act(h, xa)
                    Ho, Wo = (hH - 1) // 2 + 1, (hW - 1) // 2 + 1
                    o = pool.get(f"{tag}{bi}", (n * Ho * Wo, cout), torch.float32)
                    st, req = self._stats_req(n, cout, Ho * Wo)
                    ok = ops.conv2d_3x3(xa.view(n, hH, hW, cin), W[p + ".w"], ops.make_ep(o, bias=W[p + ".b"], gn_stats=req),
                                        stride=2)
                    h, hH, hW, hC, hst = o, Ho, Wo, cout, (st if ok else None)
                elif kind == "up":
                    xu = pool.get(f"act_up{cin}", (n * 4 * hH * hW, cin), AD)
                    ops.upsample2x_to_act(h, n, hH, hW, cin, xu)
                    hH, hW = 2 * hH, 2 * hW
                    o = pool.get(f"{tag}{bi}u", (n * hH * hW, cout), torch.float32)
                    ops.conv2d_3x3(xu.view(n, hH, hW, cin), W[p + ".w"], ops.make_ep(o, bias=W[p + ".b"]))
                    h, hC, hst = o, cout, None      # consumed by a channel concat, not by a GroupNorm
                if self.debug is not None:
                    self.debug.append((p, kind, h.detach().clone()))
            return h, hH, hW, hC, hst

        hst = None
        for bi, layers in enumerate(inp):
            h, hH, hW, hC, hst = run(layers, h, hH, hW, hC, bi, "in", hst)
            hs.append((h, hH, hW, hC))
        h, hH, hW, hC, hst = run(mid, h, hH, hW, hC, 0, "mid", hst)
        for bi, layers in enumerate(out):
            s, sH, sW, sC = hs.pop()
            if (sH, sW) != (hH, hW):
                raise ValueError(f"skip/upsample size mismatch {(sH, sW)} vs {(hH, hW)}: latent H, W must be divisible by 8")
            # the concatenated tensor regroups channels: its GroupNorm statistics cannot reuse the producers' sums, but the
            # concat pass itself can accumulate them (saves the separate statistics read of the largest fp32 tensors).
            # The consumer is a ResBlock with cin != cout (1x1 skip conv): nothing reads the concat in fp32, so it is written in
            # the 16-bit operand type only (10 instead of 20 bytes per element over concat + GroupNorm + cast).
            first = layers[0]
            if first[0] == "vrb" and first[2] != first[3]:
                cat = pool.get(f"cat16_{bi}", (n * hH * hW, hC + sC), AD)
            else:
                cat = pool.get(f"cat{bi}", (n * hH * hW, hC + sC), torch.float32)
            cst, _ = self._stats_req(n, hC + sC, hH * hW)
            ops.concat_channels(h, s, cat, stats=cst, n_img=n)
            h, hH, hW, hC, hst = run(layers, cat, hH, hW, hC + sC, bi, "out", cst)
        rows = n * hH * hW
        a = pool.get(f"act_a{hC}", (rows, hC), AD)
        self._gn(h, n, hH * hW, hC, "out.0", 1e-5, True, a, stats=hst)
        res = pool.get("net_out", (rows, 16), torch.float32)
        oc = cfg["out_channels"]
        ops.conv2d_3x3(a.view(n, hH, hW, hC), W["out.2.w"], ops.make_ep(res[:, :oc], bias=W["out.2.b"]))
        return res


# ----------------------------------------------------------------------------------------------------------------------
class VideoUNet(nn.Module):
    """Drop-in `target:` for sgm.modules.diffusionmodules.video_model.VideoUNet (constructor: video_model.py:85-120).

    Only the option set the GCD configs use is implemented (configs/infer_kubric.yaml:18-40, infer_pardom.yaml);
    anything else raises at construction instead of silently computing something different."""

    def __init__(self, in_channels, model_channels, out_channels, num_res_blocks, attention_resolutions, dropout=0.0,
                 channel_mult=(1, 2, 4, 8), conv_resample=True, dims=2, num_classes=None, use_checkpoint=False,
                 num_heads=-1, num_head_channels=-1, num_heads_upsample=-1, use_scale_shift_norm=False,
                 resblock_updown=False, transformer_depth=1, transformer_depth_middle=None, context_dim=None,
                 time_downup=False, time_context_dim=None, extra_ff_mix_layer=False, use_spatial_context=False,
                 merge_strategy="fixed", merge_factor=0.5, spatial_transformer_attn_type="softmax", video_kernel_size=3,
                 use_linear_in_transformer=False, adm_in_channels=None, aux_emb_dim=0, aux_zero_init=False,
                 disable_temporal_crossattention=False, max_ddpm_temb_period=10000):
        super().__init__()
        need = need_option("VideoUNet")
        need(dims == 2 and conv_resample and not resblock_updown and not use_scale_shift_norm, "dims/resample/updown")
        need(num_classes == "sequential" and adm_in_channels is not None, "num_classes must be 'sequential'")
        need(num_head_channels == 64, "num_head_channels must be 64")
        need(use_linear_in_transformer and extra_ff_mix_layer and use_spatial_context, "transformer layout")
        need(merge_strategy == "learned_with_images", "merge_strategy")
        need(list(video_kernel_size) == [3, 1, 1] if not isinstance(video_kernel_size, int) else False, "video_kernel_size")
        need(transformer_depth == 1 and transformer_depth_middle in (None, 1), "transformer_depth")
        need(not time_downup and not disable_temporal_crossattention and dropout == 0.0, "time_downup/dropout")
        need(max_ddpm_temb_period == 10000 and context_dim is not None, "context")
        need(model_channels % 64 == 0, "model_channels must be a multiple of 64")
        self.cfg = dict(in_channels=in_channels, out_channels=out_channels, model_channels=model_channels,
                        attention_resolutions=list(attention_resolutions), num_res_blocks=num_res_blocks,
                        channel_mult=list(channel_mult), num_head_channels=num_head_channels, transformer_depth=1,
                        context_dim=context_dim, adm_in_channels=adm_in_channels, aux_emb_dim=aux_emb_dim)
        self.in_channels, self.model_channels, self.out_channels = in_channels, model_channels, out_channels
        self.adm_in_channels, self.aux_emb_dim, self.num_classes = adm_in_channels, aux_emb_dim, num_classes
        register_param_tree(self, spec.unet_param_shapes(self.cfg))
        self._engines = EngineCache()

    def invalidate(self):
        """Forces a repack at the next forward, for in-place weight edits that weights_key cannot see."""
        self._engines.clear()

    def engine(self, device):
        return self._engines.get(self, device, lambda: UNetEngine(self.cfg, self.state_dict(), device))

    @torch.no_grad()
    def forward(self, x, timesteps, context=None, y=None, time_context=None, num_video_frames=None,
                image_only_indicator=None):
        if not x.is_cuda:
            raise RuntimeError("gcd_b200.VideoUNet runs on CUDA (sm_90a) only; there is no CPU path")
        if time_context is not None:
            raise NotImplementedError("time_context must be None (use_spatial_context=True derives it from context)")
        if image_only_indicator is not None and bool((image_only_indicator != 0).any()):
            raise NotImplementedError("image_only_indicator must be all zeros (as in every GCD call site)")
        assert (y is not None) and context is not None and num_video_frames is not None
        n, c, H, W = x.shape
        assert c == self.in_channels and y.shape[0] == n
        eng = self.engine(x.device)
        x_cl = eng.pool.get("x_cl", (n, H, W, 64), eng.AD)
        ops.nchw_to_act_nhwc(x.to(torch.float32).contiguous(), n, c, H * W, 64, x_cl)
        res = eng.forward_cl(x_cl, n, H, W, timesteps, context, y, num_video_frames)
        out = torch.empty(n, self.out_channels, H, W, device=x.device, dtype=torch.float32)
        ops.nhwc_to_nchw(res, 16, n, self.out_channels, H * W, out)
        return out.to(x.dtype)
