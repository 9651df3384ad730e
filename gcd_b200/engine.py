"""Host-side plumbing shared by the execution engines (unet.UNetEngine, vae.DecoderEngine / EncoderEngine, clip.ClipEngine) and
their drop-in modules: reference-shaped parameter trees, the packed-engine cache, named device workspaces, the GroupNorm
statistics arena and the kernel-native weight layouts."""
import importlib

import torch
import torch.nn as nn

from . import ops


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference module tree (and therefore its state_dict keys)."""


def register_param_tree(root, shapes, init=None):
    """Registers nn.Parameters under nested _Node modules so that root.state_dict() has exactly the keys of `shapes`."""
    for key, shape in shapes.items():
        parts = key.split(".")
        mod = root
        for p in parts[:-1]:
            if not hasattr(mod, p):
                mod.add_module(p, _Node())
            mod = getattr(mod, p)
        t = torch.zeros(shape) if init is None else init(key, shape)
        # requires_grad=True like any nn.Module parameter: the reference's LitEma (modules/ema.py) only shadows parameters
        # with requires_grad, and DiffusionEngine.ema_scope swaps them in with `param.data.copy_` — see weights_key()
        mod.register_parameter(parts[-1], nn.Parameter(t, requires_grad=True))


def reference_base(module, name):
    """`module.name` of the reference package when `sgm` imports (so that the reference's isinstance gates accept the drop-in
    class), else nn.Module."""
    try:
        return getattr(importlib.import_module(module), name)
    except Exception:
        return nn.Module


def need_option(who):
    """The option check of a drop-in constructor: need(cond, what) raises NotImplementedError naming `what` unless `cond`."""
    def need(cond, what):
        if not cond:
            raise NotImplementedError(f"gcd_b200.{who}: unsupported option ({what}); only the GCD configs are built")
    return need


def weights_key(module, device):
    """Cache key of a drop-in module's packed engine: (data_ptr, _version) of every parameter PLUS a content probe of nine
    tensors spread over the parameter list. `_version` alone misses `param.data.copy_(...)` — exactly what the reference's
    LitEma.copy_to / restore do (modules/ema.py) — so an EMA swap would otherwise keep running the stale packed weights.
    Costs one small device->host read per engine() call (once per sample on the fused path)."""
    ps = list(module.parameters())
    meta = tuple((p.data_ptr(), p._version) for p in ps)
    probe = ps[::max(1, len(ps) // 8)][:8] + [ps[-1]]
    vals = torch.stack([p.detach().reshape(-1)[:512].double().sum().cpu() for p in probe]).tolist()
    return (str(device), meta, tuple(vals))


class EngineCache:
    """The packed engine(s) of a drop-in module. Weights may be (re)loaded at any time (init_from_ckpt, EMA swap through
    `.data.copy_`): the engines are rebuilt lazily when any parameter of `module` changed (weights_key); clear() forces it for
    in-place edits the key cannot see. Up to `slots` engines over the same weights are kept, one per `extra` key; a weight change
    drops them all. Old engines are dropped BEFORE a new one is built, so two packed weight sets are never alive at once."""

    def __init__(self, slots=1):
        self.slots = slots
        self.clear()

    def clear(self):
        self.key, self.engines = None, {}

    def get(self, module, device, build, extra=None):
        key = weights_key(module, device)
        if key != self.key:
            self.clear()
            self.key = key
        if extra not in self.engines:
            if len(self.engines) >= self.slots:
                self.engines.pop(next(iter(self.engines)))
            self.engines[extra] = build()
        return self.engines[extra]


class BufferPool:
    """Named device workspaces, allocated once per (name, shape, dtype) and reused across blocks and steps."""

    def __init__(self, device):
        self.device = device
        self.bufs = {}

    def get(self, name, shape, dtype):
        key = (name, tuple(shape), dtype)
        b = self.bufs.get(key)
        if b is None:
            b = torch.empty(shape, device=self.device, dtype=dtype)
            self.bufs[key] = b
        return b

    def nbytes(self):
        return sum(b.numel() * b.element_size() for b in self.bufs.values())

    def release(self, name):
        """Drops the workspaces named `name` (their memory returns to the caching allocator)."""
        self.bufs = {k: b for k, b in self.bufs.items() if k[0] != name}

    def release_rows(self, rows):
        """Drops the workspaces whose leading dimension is `rows` (their memory returns to the caching allocator)."""
        self.bufs = {k: b for k, b in self.bufs.items() if k[1][:1] != (rows,)}


class StatsArena:
    """float64 scratch for the GroupNorm statistics that tensor-core epilogues accumulate (gcd_epilogue.gn_stats): one slot per
    producer -> consumer hand-off of a forward pass, the WHOLE arena zeroed by one memset at the start of the pass (round 1
    zeroed a ring buffer before each of the ~130 producers: ~130 extra launches per CFG forward, 2 % of its time in the `elem`
    class of tools/prof_forward.py)."""
    SLOTS = 256

    def __init__(self, pool):
        self.pool, self.slot, self.buf, self.i = pool, 0, None, 0

    def reset(self, n_img):
        """n_img: the largest number of images (frames) any statistics of this pass are kept for."""
        need = max(n_img, 64) * 64
        if need > self.slot:
            self.slot = need
            self.buf = self.pool.get("gn_arena", (self.SLOTS * need,), torch.float64)
        self.i = 0
        ops.zero_tensor(self.buf)

    def take(self, n_img):
        need = max(n_img, 64) * 64
        assert need <= self.slot and self.i < self.SLOTS, "GroupNorm statistics arena exhausted"
        st = self.buf[self.i * self.slot:(self.i + 1) * self.slot]
        self.i += 1
        return st


class Engine:
    """Packed weights `w` (16-bit GEMM operands, fp32 biases and norm parameters), AlphaBlender factors `alpha`, workspaces and
    GroupNorm statistics arena of one network on one device.

    The packers take `src`: a key prefix of the state dict `sd` (`<src>.weight`, `<src>.bias`) or a (weight, bias) pair of
    tensors, and store `<name>.w` / `<name>.b` (norms: `<name>.g` / `<name>.b`)."""

    def __init__(self, device):
        self.device = torch.device(device)
        self.AD = ops.act_dtype()
        self.pool = BufferPool(self.device)
        self.arena = StatsArena(self.pool)
        self.w, self.alpha = {}, {}

    # ------------------------------------------------------------------------------------------------ weight packing
    def _f32(self, t):
        return t.detach().to(self.device, torch.float32)

    def _put(self, sd, name, src, pack):
        w, b = (sd[src + ".weight"], sd.get(src + ".bias")) if isinstance(src, str) else src
        self.w[name + ".w"] = pack(self._f32(w)).to(self.AD).contiguous()
        if b is not None:
            self.w[name + ".b"] = self._f32(b).contiguous()

    def _conv3(self, sd, name, src, cin_pad=None):
        """3x3 conv [Co, Ci, 3, 3] -> [Co, (ky, kx, c)], the input channels zero-padded to `cin_pad`."""
        def pack(w):
            if cin_pad is not None and cin_pad != w.shape[1]:
                w = torch.cat([w, w.new_zeros(w.shape[0], cin_pad - w.shape[1], 3, 3)], 1)
            return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)
        self._put(sd, name, src, pack)

    def _convt(self, sd, name, src):
        """(3,1,1) temporal conv [Co, Ci, 3, 1, 1] -> [Co, (kt, c)]."""
        self._put(sd, name, src, lambda w: w[:, :, :, 0, 0].permute(0, 2, 1).reshape(w.shape[0], -1))

    def _lin(self, sd, name, src):
        """Linear [Co, Ci] or 1x1 conv [Co, Ci, 1, 1] -> [Co, Ci]; the bias is optional."""
        self._put(sd, name, src, lambda w: w.reshape(w.shape[0], -1))

    def _norm(self, sd, name, src):
        self.w[name + ".g"] = self._f32(sd[src + ".weight"]).contiguous()
        self.w[name + ".b"] = self._f32(sd[src + ".bias"]).contiguous()

    # ------------------------------------------------------------------------------------------------ GroupNorm
    def _gn(self, x, n_img, rows, C, name, eps, silu, out, stats=None):
        """GroupNorm(32) (+SiLU) -> act. `stats`: statistics already accumulated by the producing tensor-core op."""
        st = stats if stats is not None else self.pool.get("gn_stats", (max(n_img, 64) * 64,), torch.float64)
        ops.groupnorm(x, n_img, rows, C, self.w[name + ".g"], self.w[name + ".b"], eps, silu, out, st,
                      have_stats=stats is not None)

    def _stats_req(self, n_img, C, rows_per_img):
        """Zeroed float64 statistics slot (StatsArena, zeroed once per forward) + the epilogue descriptor."""
        st = self.arena.take(n_img)
        return st, (st, C // 32, 32, rows_per_img)
