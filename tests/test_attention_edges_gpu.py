"""Attention at production sizes and at the inputs where it goes wrong, against float64 from the same 16-bit inputs.

Four paths compute softmax(q k^T / sqrt(d)) v:
- UNet spatial: attn_spatial.cu (wgmma flash attention, d = 64);
- UNet temporal: attn_temporal.cu, the persistent mma.sync kernel for T <= 16 and the fp32 CUDA-core kernel above;
- the CLIP tower: clip.cu attn_d80_kernel (d = 80);
- the VAE's mid AttnBlock: vae._VAEEngine._attn (bmm_nt scores in fp32, softmax_rows, bmm_nt P.V^T with the v bias).

Each packs its softmax weights P to the 16-bit operand type for the P.V product. fp16 flushes anything below 2^-25 to zero, so a
row whose dominant key has |v| ~ 0 and whose other keys sit 17.4-18 nats below it with |v| of order 1-4 ("planted" rows) loses
most of its output unless P is packed with an offset (2^15 P; oracle/error_model.py, attention_scale). The temporal kernel for
T > 16 keeps P in fp32: its planted rows are the control showing the reference is right.

Every check is EM.check: |y - ref| <= u_out |ref| + eta + kappa 2^-24 scale, per element.
"""
import math

import pytest
import torch

from oracle import error_model as EM

gpu = pytest.mark.gpu
F16 = torch.float16

# UNet token counts and head counts per level (channels 320 / 640 / 1280 / 1280, head_dim 64) of a 72x128 and a 32x48 latent
LEVELS_72x128 = [(9216, 5), (2304, 10), (576, 20), (144, 20)]
LEVELS_32x48 = [(1536, 5), (384, 10), (96, 20), (24, 20)]
TEMPORAL_BLOCK = 4 * 6          # warps per block x resident blocks per SM of attn_temporal_mma_kernel's persistent grid


@pytest.fixture(scope="module")
def ops():
    from gcd_b200 import ops as o
    o.lib()
    return o


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def sdpa64(q, k, v, scale):
    """float64 softmax(q k^T * scale) v over the last two dims, with the error model's terms: sum_j p_j |v_j| and
    p_max * sum_j |v_j| (the subnormal-P term of the flash kernels)."""
    q, k, v = q.double(), k.double(), v.double()
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, -1)
    va = v.abs()
    return p @ v, p @ va, p.amax(-1, keepdim=True) * va.sum(-2, keepdim=True)


def spatial_ref(qkv, frames, tokens, heads, d=64, chunk=2048):
    """[frames, tokens, 3 * heads * d] -> (ref, pv, cv) as [frames, tokens, heads * d], chunked over queries."""
    C = heads * d
    q, k, v = qkv.view(frames, tokens, 3, heads, d).permute(2, 0, 3, 1, 4)
    outs = [torch.empty(frames, tokens, C, dtype=torch.float64, device=qkv.device) for _ in range(3)]
    for i in range(0, tokens, chunk):
        for o, r in zip(outs, sdpa64(q[:, :, i:i + chunk], k, v, d ** -0.5)):
            o[:, i:i + chunk] = r.permute(0, 2, 1, 3).reshape(frames, -1, C)
    return outs


def temporal_ref(qkv, clips, T, tokens, heads, chunk=1024):
    """[clips * T, tokens, 3 * heads * 64] -> (ref, pv, cv) as [clips * T, tokens, heads * 64]: attention over the T frames of
    each (clip, position, head), chunked over positions."""
    C = heads * 64
    x = qkv.view(clips, T, tokens, 3, heads, 64)
    outs = [torch.empty(clips, T, tokens, C, dtype=torch.float64, device=qkv.device) for _ in range(3)]
    for s0 in range(0, tokens, chunk):
        q, k, v = x[:, :, s0:s0 + chunk].permute(3, 0, 2, 4, 1, 5)          # [clips, s, heads, T, 64]
        for o, r in zip(outs, sdpa64(q, k, v, 0.125)):
            o[:, :, s0:s0 + chunk] = r.permute(0, 3, 1, 2, 4).reshape(clips, T, -1, C)
    return [o.view(clips * T, tokens, C) for o in outs]


def check_attention(out, ref, pv, cv, AD, name):
    return EM.check(out, ref, EM.attention_scale(pv, AD, v_abs=cv), "attention", name)


def temporal_grid_warps(ops, clips, tokens, heads):
    """Warps of attn_temporal_mma_kernel's persistent grid (gcd_attention_temporal): min(groups / 4 blocks, 6 per SM) x 4."""
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    groups = clips * tokens * heads
    return groups, 4 * min((groups + 3) // 4, 6 * n_sm), n_sm


def run_temporal(ops, qkv, clips, T, tokens, heads):
    out = torch.empty(clips * T, tokens, heads * 64, device="cuda", dtype=qkv.dtype)
    ops.attention_temporal(qkv, clips, T, tokens, heads, out)
    return out


# ---------------------------------------------------------------------------------------------------------- planted rows
PLANT_TOP = 20.0     # logit of the dominant key
PLANT_GAP = (17.4, 18.0)   # below it: past fp16's flush threshold 2^-25 = e^-17.33 (closer keys round up to 2^-24 instead)


def planted_logits(shape, dom, g):
    """Logits [..., keys]: PLANT_TOP at key dom[...] (a tensor of shape[:-1]), PLANT_TOP - U(PLANT_GAP) elsewhere."""
    lo, hi = PLANT_GAP
    s = PLANT_TOP - lo - (hi - lo) * torch.rand(shape, generator=g, device=g.device, dtype=torch.float64)
    s.scatter_(-1, dom.unsqueeze(-1), PLANT_TOP)
    return s


def planted_values(keys, d, dom, g):
    """Values [..., keys, d]: |v| ~ 1e-3 at the dominant key dom[...], sign(channel) * U(1, 4) elsewhere (one sign per
    channel, so that the mass of the other keys adds up in the output)."""
    lead = dom.shape
    v = 1.0 + 3.0 * torch.rand(*lead, keys, d, generator=g, device=g.device, dtype=torch.float64)
    sign = torch.where(torch.rand(*lead, 1, d, generator=g, device=g.device) < 0.5, -1.0, 1.0).double()
    v = v * sign
    small = 1e-3 * torch.randn(*lead, 1, d, generator=g, device=g.device, dtype=torch.float64)
    v.scatter_(-2, dom[..., None, None].expand(*lead, 1, d), small)
    return v


def simulate_packed_p(s, v, offset, dtype=F16):
    """The flash kernels' P arithmetic on one block of logits s [..., keys] (natural log units) and values v [..., keys, d]:
    e = exp(s - max) in fp32, P = offset * e packed to `dtype`, O = sum_j P_j v_j and l = offset * sum_j e_j, O / l in fp32."""
    s32 = s.float()
    e = torch.exp(s32 - s32.amax(-1, keepdim=True))
    p16 = (e * offset).to(dtype)
    o = p16.double().unsqueeze(-2) @ v.double()
    l = (e.sum(-1, keepdim=True) * offset).double().unsqueeze(-1)
    return (o / l).squeeze(-2).float()


@pytest.mark.parametrize("keys", [14, 257, 9216])
def test_packed_p_offset_error_model(keys):
    """CPU: the P arithmetic of the flash kernels on planted rows, packed to fp16 without and with the 2^15 offset. Without it the
    error exceeds the relative-only bound (u_act sum p |v|) by two orders of magnitude, and the subnormal term for the offset
    P (2^-40 p_max sum |v|) does not cover it; with it the output is inside the bound with the subnormal term."""
    g = torch.Generator().manual_seed(keys)
    rows, d = 32, 64
    dom = torch.randint(0, keys, (rows,), generator=g)
    s = planted_logits((rows, keys), dom, g)
    v = planted_values(keys, d, dom, g).to(F16).double()          # 16-bit values, as the kernels read them
    p = torch.softmax(s, -1)
    ref = (p.unsqueeze(-2) @ v).squeeze(-2)
    pv = (p.unsqueeze(-2) @ v.abs()).squeeze(-2)
    cv = p.amax(-1, keepdim=True) * v.abs().sum(-2)
    kappa = EM.KAPPA["attention"]
    ratio = lambda y, sc: ((y.double() - ref).abs() / (kappa * EM.EPS32 * sc)).max().item()   # fp32 output: u_out = eta = 0

    plain = simulate_packed_p(s, v, 1.0)
    r_old = ratio(plain, EM.attention_scale(pv, F16))
    r_new = ratio(plain, EM.attention_scale(pv, F16, v_abs=cv))
    shifted = simulate_packed_p(s, v, EM.P_OFFSET)
    r_fix = ratio(shifted, EM.attention_scale(pv, F16, v_abs=cv))
    print(f"planted rows, {keys} keys: error/bound without offset {r_old:.1f} (with the subnormal term {r_new:.1f}), "
          f"with 2^15 offset {r_fix:.3f}")
    assert r_old > 50 and r_new > 50, (r_old, r_new)
    assert r_fix < 0.25, r_fix
    EM.check(shifted, ref, EM.attention_scale(pv, F16, v_abs=cv), "attention", f"simulated offset P, {keys} keys")
    # bf16 keeps fp32's exponent: no offset needed
    EM.check(simulate_packed_p(s, v, 1.0, torch.bfloat16), ref, EM.attention_scale(pv, torch.bfloat16, v_abs=cv), "attention",
             f"simulated bf16 P, {keys} keys")


def plant_qkv(logits, v, d, qk_dim0):
    """Per head: q = (qk_dim0, 0, ...), k = (logit * sqrt(d) / qk_dim0, noise...), so that q.k / sqrt(d) = the planted logit (up to
    the 16-bit rounding of k, which the float64 reference sees as well). logits [..., heads, keys], v [..., heads, keys, d];
    returns q, k, v as [..., keys, heads, d]."""
    g = gen(int(logits.numel()) % 100003)
    k = 0.5 * torch.randn(*v.shape, generator=g, device="cuda", dtype=torch.float64)
    k[..., 0] = logits * (d ** 0.5 / qk_dim0)
    q = torch.zeros_like(k)
    q[..., 0] = qk_dim0
    return [t.transpose(-3, -2) for t in (q, k, v)]


@gpu
@pytest.mark.parametrize("where", ["first", "last"])
def test_spatial_planted_subnormal_p(ops, where):
    """9216 tokens, one frame. 'first': the dominant key is in the first key block, so every later block packs P against the
    established maximum. 'last': it is in the last block; the earlier blocks are packed against their own maximum and rescaled
    in fp32, and the other keys of the last block have v = 0 (in-kernel control)."""
    AD = ops.act_dtype()
    frames, tokens, heads, d = 1, 9216, 5, 64
    g = gen(11 if where == "first" else 12)
    lo = 0 if where == "first" else tokens - 64
    dom = torch.randint(lo, lo + 64, (frames, heads), generator=g, device="cuda")
    logits = planted_logits((frames, heads, tokens), dom, g)
    v = planted_values(tokens, d, dom, g)
    if where == "last":
        keep = v[..., lo:, :].clone()
        v[..., lo:, :] = 0
        v.scatter_(-2, dom[..., None, None].expand(frames, heads, 1, d), keep.gather(-2, (dom - lo)[..., None, None].expand(
            frames, heads, 1, d)))
    q, k, v = plant_qkv(logits, v, d, 8.0)
    qkv = torch.cat([t.reshape(frames, tokens, heads * d) for t in (q, k, v)], -1).to(AD).contiguous()
    out = torch.empty(frames, tokens, heads * d, device="cuda", dtype=AD)
    ops.attention_spatial(qkv, frames, tokens, heads, out)
    ref, pv, cv = spatial_ref(qkv, frames, tokens, heads)
    check_attention(out, ref, pv, cv, AD, f"attention_spatial planted rows, dominant key in the {where} block")


@gpu
def test_d80_planted_subnormal_p(ops):
    """The CLIP tower's 257 tokens, dominant key in the first key block."""
    AD = ops.act_dtype()
    n, L, heads, d = 2, 257, 16, 80
    g = gen(13)
    dom = torch.randint(0, 64, (n, heads), generator=g, device="cuda")
    logits = planted_logits((n, heads, L), dom, g)
    v = planted_values(L, d, dom, g)
    q, k, v = plant_qkv(logits, v, d, 9.0)
    qkv = torch.cat([t.reshape(n * L, heads * d) for t in (q, k, v)], -1).to(AD).contiguous()
    out = torch.empty(n * L, heads * d, device="cuda", dtype=AD)
    ops.attention_d80(qkv, n, L, heads, out)
    ref, pv, cv = spatial_ref(qkv.view(n, L, -1), n, L, heads, d=d)
    check_attention(out.view(n, L, -1), ref, pv, cv, AD, "attention_d80 planted rows")


def planted_temporal_qkv(clips, T, tokens, heads, AD, seed):
    g = gen(seed)
    dom = torch.randint(0, T, (clips, tokens, heads), generator=g, device="cuda")
    logits = planted_logits((clips, tokens, heads, T), dom, g)
    v = planted_values(T, 64, dom, g)                                  # [clips, tokens, heads, T, 64]
    q, k, v = plant_qkv(logits, v, 64, 8.0)                     # [clips, tokens, T, heads, 64]
    qkv = torch.cat([t.permute(0, 2, 1, 3, 4).reshape(clips, T, tokens, heads * 64) for t in (q, k, v)], -1)
    return qkv.reshape(clips * T, tokens, 3 * heads * 64).to(AD).contiguous()


@gpu
@pytest.mark.parametrize("T", [14, 25])
def test_temporal_planted_subnormal_p(ops, T):
    """T = 14: the mma.sync kernel packs P to 16 bits. T = 25: the CUDA-core kernel keeps P in fp32 (control)."""
    AD = ops.act_dtype()
    clips, tokens, heads = 2, 2304, 10
    qkv = planted_temporal_qkv(clips, T, tokens, heads, AD, seed=T)
    out = run_temporal(ops, qkv, clips, T, tokens, heads)
    ref, pv, cv = temporal_ref(qkv, clips, T, tokens, heads)
    check_attention(out, ref, pv, cv, AD, f"attention_temporal planted rows T={T}")


def vae_pv(ops, sc, scale, vt, bias, pr, o):
    """The VAE mid attention's P.V chain as vae._VAEEngine._attn runs it: P_SCALE * softmax_rows, then bmm_nt against V^T with
    the bias P_SCALE * b_v and a_acc = 1 / P_SCALE."""
    from gcd_b200 import vae
    n, S = vt.shape[0], vt.shape[2]
    ops.softmax_rows(sc, scale, pr, out_scale=vae.P_SCALE)
    ops.bmm_nt(pr.view(n, S, S), vt, ops.make_ep(o, bias=bias * vae.P_SCALE, a_acc=1.0 / vae.P_SCALE))


def softmax_pv_scale(arg, p, vt, bias, AD, arg_err=None):
    """Scale of o = softmax(arg) (v + b) as softmax_rows + bmm_nt compute it, for one frame; arg [S, S] float64, p its softmax,
    vt [C, S]. In units of 2^-24 with kappa = attention:
    - softmax_rows: p_j (1 + eps_j), |eps_j| of order (1 + |arg_j| + arg_err_j) 2^-24, moves o by sum_j p_j |eps_j| (|v_j| + |o_v|);
    - P packed to 16 bits: attention_scale with c = 1 (softmax_rows' P is normalised);
    - the P.V GEMM: 2 (sum_j p_j |v_j| + |b|) (tc_gemm's kappa is twice attention's); its k-loop term is passed to EM.check apart.
    arg_err: the error of the exponent's argument carried over from the score GEMM, in units of 2^-24."""
    v = vt.double().t()
    va = v.abs()
    w = 1.0 + arg.abs() if arg_err is None else 1.0 + arg.abs() + arg_err
    pw = p * w
    ov = (p @ v).abs()
    pv = p @ va
    s = pw @ va + pw.sum(-1, keepdim=True) * ov
    s = s + EM.attention_scale(pv, AD, v_abs=va.sum(0, keepdim=True), c=1.0)
    return s + 2.0 * (pv + bias.double().abs())


@gpu
def test_vae_chain_planted_subnormal_p(ops):
    """softmax_rows followed by bmm_nt with the v bias at the VAE's 9216 x 9216 scores and C = 512; the scores are planted."""
    AD = ops.act_dtype()
    S, C = 9216, 512
    scale = C ** -0.5
    g = gen(17)
    keys = torch.randperm(S, generator=g, device="cuda")[:64]                 # the keys that dominate a row, |v| ~ 0
    dom = keys[torch.randint(0, 64, (S,), generator=g, device="cuda")]
    sc = (planted_logits((S, S), dom, g) / scale).float()
    v = planted_values(S, C, keys[:1], g)[0]
    v[keys] = 1e-3 * torch.randn(64, C, generator=g, device="cuda", dtype=torch.float64)
    vt = v.t().contiguous().to(AD).unsqueeze(0)
    bias = 1e-3 * torch.randn(C, generator=g, device="cuda")
    pr = torch.empty(S, S, device="cuda", dtype=AD)
    o = torch.empty(S, C, device="cuda", dtype=AD)
    vae_pv(ops, sc, scale, vt, bias, pr, o)
    arg = (sc.double() - sc.double().amax(-1, keepdim=True)) * scale
    p = torch.softmax(arg, -1)
    ref = p @ vt[0].double().t() + bias.double()
    EM.check(o, ref, softmax_pv_scale(arg, p, vt[0], bias, AD), "attention", "VAE softmax_rows + P.V planted rows",
             steps=EM.gemm_step_sums(p, vt[0]))


# ---------------------------------------------------------------------------------------------------------- temporal
@gpu
@pytest.mark.parametrize("clips", [2, 4])
@pytest.mark.parametrize("tokens,heads", LEVELS_72x128 + LEVELS_32x48)
def test_temporal_production_groups(ops, clips, tokens, heads):
    """T = 14 at every UNet level of a 72x128 and a 32x48 latent, one sample (2 clips: CFG) and two (4 clips). At the level-1
    shapes every warp of the persistent grid walks many groups, with the next group's loads in flight."""
    AD = ops.act_dtype()
    T = 14
    groups, nwarps, n_sm = temporal_grid_warps(ops, clips, tokens, heads)
    if tokens in (9216, 1536):
        assert groups > TEMPORAL_BLOCK * n_sm and nwarps == TEMPORAL_BLOCK * n_sm, (groups, nwarps, n_sm)
    print(f"temporal {clips}x{T}x{tokens}x{heads}: {groups} groups over {nwarps} warps, {math.ceil(groups / nwarps)} trips, "
          f"last trip {groups - (math.ceil(groups / nwarps) - 1) * nwarps} groups")
    g = gen(tokens * heads + clips)
    qkv = (1.5 * torch.randn(clips * T, tokens, 3 * heads * 64, generator=g, device="cuda")).to(AD)
    out = run_temporal(ops, qkv, clips, T, tokens, heads)
    ref, pv, cv = temporal_ref(qkv, clips, T, tokens, heads)
    check_attention(out, ref, pv, cv, AD, f"attention_temporal {clips}x{T}x{tokens}x{heads}")


@gpu
def test_temporal_ragged_last_trip(ops):
    """3 full trips of the persistent grid plus at most 10 groups, whatever the SM count."""
    AD = ops.act_dtype()
    clips, T, heads = 2, 14, 5
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    tokens = 3 * TEMPORAL_BLOCK * n_sm // (clips * heads) + 1
    groups, nwarps, _ = temporal_grid_warps(ops, clips, tokens, heads)
    assert nwarps == TEMPORAL_BLOCK * n_sm and groups % nwarps and groups // nwarps == 3, (groups, nwarps)
    g = gen(23)
    qkv = (1.5 * torch.randn(clips * T, tokens, 3 * heads * 64, generator=g, device="cuda")).to(AD)
    out = run_temporal(ops, qkv, clips, T, tokens, heads)
    ref, pv, cv = temporal_ref(qkv, clips, T, tokens, heads)
    check_attention(out, ref, pv, cv, AD, f"attention_temporal ragged last trip ({groups} groups, {nwarps} warps)")


@gpu
@pytest.mark.parametrize("T", [1, 2, 8, 15, 16, 17, 25, 32])
def test_temporal_T_edges(ops, T):
    """Both kernels and the switch between them (T <= 16: mma.sync; above: fp32 CUDA cores); 4000 groups, more than one trip."""
    AD = ops.act_dtype()
    clips, tokens, heads = 2, 400, 5
    g = gen(100 + T)
    qkv = (1.5 * torch.randn(clips * T, tokens, 3 * heads * 64, generator=g, device="cuda")).to(AD)
    out = run_temporal(ops, qkv, clips, T, tokens, heads)
    ref, pv, cv = temporal_ref(qkv, clips, T, tokens, heads)
    check_attention(out, ref, pv, cv, AD, f"attention_temporal T={T}")


@gpu
@pytest.mark.parametrize("T", [0, 33])
def test_temporal_T_out_of_range(ops, T):
    from gcd_b200 import _lib
    AD = ops.act_dtype()
    qkv = torch.zeros(2 * max(T, 1), 16, 3 * 64, device="cuda", dtype=AD)
    out = torch.zeros(2 * max(T, 1), 16, 64, device="cuda", dtype=AD)
    n0 = ops.launch_count()
    with pytest.raises(_lib.GcdError, match="unsupported"):
        ops.attention_temporal(qkv, 2, T, 16, 1, out)
    assert ops.launch_count() == n0


def peaked_temporal_qkv(clips, T, tokens, heads, AD, kind, seed):
    """kind 'logit100': |logits| up to ~100. 'tie': keys i1 != i2 of every group are equal and >= 30 nats above the others for
    every query. 'onehot': one key >= 100 nats above the others. Returns qkv and, for tie / onehot, the dominant keys [clips, tokens,
    heads, 2]."""
    g = gen(seed)
    x = torch.randn(clips, T, tokens, 3, heads, 64, generator=g, device="cuda")
    if kind == "logit100":
        x[:, :, :, :2] *= 4.7
        return x.reshape(clips * T, tokens, -1).to(AD), None
    i1 = torch.randint(0, T, (clips, tokens, heads), generator=g, device="cuda")
    i2 = (i1 + torch.randint(1, max(T, 2), (clips, tokens, heads), generator=g, device="cuda")) % T if kind == "tie" else i1
    u = torch.randn(clips, 1, tokens, heads, 64, generator=g, device="cuda")
    u = 8.0 * u / u.norm(dim=-1, keepdim=True)                      # |u|^2 = 64: q.u / 8 = 8 a for q = a u
    k = x[:, :, :, 1]                                               # a view: the keys are planted in place
    a, k_scale = (6.0, 0.25) if kind == "tie" else (16.0, 0.1)      # top logit 48 / 128, the others' spread a k_scale
    x[:, :, :, 0] = a * u + 0.1 * x[:, :, :, 0]
    k *= k_scale
    for i in (i1, i2):
        k.scatter_(1, i[:, None, :, :, None].expand(clips, 1, tokens, heads, 64), u)
    return x.reshape(clips * T, tokens, -1).to(AD), torch.stack([i1, i2], -1)


@gpu
@pytest.mark.parametrize("T", [14, 25])
@pytest.mark.parametrize("kind", ["logit100", "tie", "onehot"])
def test_temporal_peaked_rows(ops, T, kind):
    AD = ops.act_dtype()
    clips, tokens, heads = 2, 576, 20
    qkv, dom = peaked_temporal_qkv(clips, T, tokens, heads, AD, kind, seed=T * 7 + len(kind))
    out = run_temporal(ops, qkv, clips, T, tokens, heads)
    ref, pv, cv = temporal_ref(qkv, clips, T, tokens, heads)
    name = f"attention_temporal {kind} T={T}"
    x = qkv.view(clips, T, tokens, 3, heads, 64)
    s = torch.einsum("atshd,aushd->ashtu", x[:, :, :, 0].double(), x[:, :, :, 1].double()) * 0.125   # [clips, s, h, tq, tk]
    if kind == "logit100":
        assert s.abs().max().item() > 80, s.abs().max().item()
    check_attention(out, ref, pv, cv, AD, name)
    if kind == "logit100":
        return
    v = x[:, :, :, 2].permute(0, 2, 3, 1, 4)                                     # [clips, s, h, T, 64]
    vd = torch.stack([v.gather(3, dom[..., j, None, None].expand(clips, tokens, heads, 1, 64))[..., 0, :]
                      for j in range(2)], -2).double()                           # [clips, s, h, 2, 64]
    top = s.gather(-1, dom[:, :, :, None, :1].expand(clips, tokens, heads, T, 1))
    rest = s.scatter(-1, dom[:, :, :, None, :].expand(clips, tokens, heads, T, 2), -math.inf).amax(-1, keepdim=True)
    gap = (top - rest).min().item()
    want = vd.mean(-2)[:, None].expand(clips, T, tokens, heads, 64).reshape(clips * T, tokens, heads * 64)
    # ties: the output is the mean of the two values; one-hot: it is v_j. Beyond the output's rounding, the bound allows twice
    # the exact distance of the softmax from that: the mass of the other keys (< e^-gap sum |v|), with room for its own fp32
    # rounding. It matters only where the mean is ~0 and the 16-bit type's eta is below it (bf16)
    assert gap >= (30 if kind == "tie" else 100), gap
    EM.check(out, want, 2.0 * (ref - want).abs() / (EM.KAPPA["attention"] * EM.EPS32), "attention", name + " vs v")
    if kind == "onehot":
        exact = torch.equal(out, want.to(AD))
        print(f"{name}: bit-exact v_j: {exact}")
        assert exact


# ---------------------------------------------------------------------------------------------------------- VAE AttnBlock
def vae_attn_state(C, seed):
    """AttnBlock state dict with Wq = Wk so that every query peaks on its own key (q.k / sqrt(C) ~ 50 on the diagonal, ~40 nats
    above the rest), and a v bias several times |v|."""
    g = torch.Generator().manual_seed(seed)
    w = lambda s: torch.randn(C, C, 1, 1, generator=g) * s
    wq = w(0.066)
    sd = {"norm.weight": 1 + 0.1 * torch.randn(C, generator=g), "norm.bias": 0.1 * torch.randn(C, generator=g),
          "q.weight": wq, "q.bias": 0.02 * torch.randn(C, generator=g),
          "k.weight": wq.clone(), "k.bias": 0.02 * torch.randn(C, generator=g),
          "v.weight": w(C ** -0.5), "v.bias": 4.0 * torch.randn(C, generator=g),
          "proj_out.weight": w(C ** -0.5), "proj_out.bias": 0.1 * torch.randn(C, generator=g)}
    return {f"mid.attn_1.{k}": t for k, t in sd.items()}


@gpu
@pytest.mark.parametrize("S,n", [(9216, 8), (1536, 14), (24, 3)])
def test_vae_mid_attention_stages(ops, S, n):
    """vae._VAEEngine._attn, stage by stage against float64 from the engine's own 16-bit intermediates. At S = 9216 the fp32 scores
    of 7 frames fit one chunk, so 8 frames run as 7 + 1."""
    from gcd_b200 import vae
    AD = ops.act_dtype()
    C, p, rows = 512, "mid.attn_1", n * S
    eng = vae._VAEEngine({}, [], "cuda")
    sd = vae_attn_state(C, seed=S + n)
    eng._pack_attn(sd, p)
    g = gen(S * n)
    x0 = 0.5 + torch.randn(rows, C, generator=g, device="cuda")
    x = x0.clone()
    eng._attn(p, x, C, n, S)
    torch.cuda.synchronize()
    buf = lambda name, shape: eng.pool.bufs[(name, tuple(shape), AD)]
    a, q, k = buf(f"a{C}_{rows}", (rows, C)), buf("attn_q", (rows, C)), buf("attn_k", (rows, C))
    vt, o = buf("attn_vt", (n, C, S)), buf("attn_o", (rows, C))
    W = {key: t.cuda().double().reshape(t.shape[0], -1) if t.dim() > 1 else t.cuda().double()
         for key, t in ((k_[len(p) + 1:], t) for k_, t in sd.items())}
    w16 = lambda name: eng.w[f"{p}.{name}.w"]
    # GroupNorm(32, eps 1e-6)
    xr = x0.double().view(n, S, 32, C // 32)
    mean = xr.mean((1, 3), keepdim=True)
    rstd = (xr.var((1, 3), unbiased=False, keepdim=True) + 1e-6).rsqrt()
    gg, bb = W["norm.weight"].view(32, -1), W["norm.bias"].view(32, -1)
    ref = ((xr - mean) * rstd * gg + bb).view(rows, C)
    EM.check(a, ref, ((xr.abs() + mean.abs()) * rstd * gg.abs() + bb.abs()).view(rows, C), "norm", f"VAE attn {n}x{S} GroupNorm")
    del xr, ref
    # q, k, v^T
    for name, t in (("q", q), ("k", k)):
        EM.check(t, a.double() @ w16(name).double().t() + W[f"{name}.bias"], EM.gemm_scale(a, w16(name), W[f"{name}.bias"]),
                 "gemm", f"VAE attn {n}x{S} {name}")
    for f in range(n):
        af = a[f * S:(f + 1) * S]
        EM.check(vt[f], w16("v").double() @ af.double().t(), EM.gemm_scale(w16("v"), af), "gemm", f"VAE attn {n}x{S} v^T {f}")
    # o = softmax(q k^T / sqrt(C)) (v + b_v), per frame
    scale = C ** -0.5
    peak = 0.0
    for f in range(n):
        qf, kf = q[f * S:(f + 1) * S].double(), k[f * S:(f + 1) * S].double()
        sc = qf @ kf.t()
        gs = qf.abs() @ kf.abs().t()                                  # the score GEMM's scale
        arg = (sc - sc.amax(-1, keepdim=True)) * scale
        peak = max(peak, (sc * scale).abs().max().item())
        # error of the exponent's argument from the score GEMM, (32 + GEMM_STEP K / 16) 2^-24 (g_j + g_max) scale at most
        # (tc_gemm's kappa and its k-loop term with every running sum at g), in units of kappa_attention 2^-24
        gmax = gs.gather(-1, sc.argmax(-1, keepdim=True))
        arg_err = (EM.KAPPA["gemm"] + EM.GEMM_STEP * C / 16) / EM.KAPPA["attention"] * scale * (gs + gmax)
        del sc, gs
        pf = torch.softmax(arg, -1)
        ref = pf @ vt[f].double().t() + W["v.bias"]
        sf = softmax_pv_scale(arg, pf, vt[f], eng.w[p + ".v.b"], AD, arg_err=arg_err)
        del arg, arg_err
        EM.check(o[f * S:(f + 1) * S], ref, sf, "attention", f"VAE attn {n}x{S} softmax P.V frame {f}",
                 steps=EM.gemm_step_sums(pf, vt[f]))
        del pf, ref, sf
    assert peak > 40, peak
    # x + proj_out(o)
    Wp = w16("proj_out")
    EM.check(x, x0.double() + o.double() @ Wp.double().t() + W["proj_out.bias"], EM.gemm_scale(o, Wp, W["proj_out.bias"], x0),
             "gemm", f"VAE attn {n}x{S} x + proj_out(o)")
