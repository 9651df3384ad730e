"""GPU tests of the conditioner's OpenCLIP ViT-H/14 image tower and of GCDHotPath.condition: the new kernels against fp32 torch,
the whole tower and the (c, uc) conditioning against stored goldens (tests/golden/clip_*.pt, cond_*.pt: the reference's
embedder / conditioner code over an fp32 restatement of open_clip and kornia, see DESIGN.md §4)."""
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

# Per-frame rel-L2 of the pooled, projected embedding vs the fp32 golden (fp16 operands, fp32 accumulation / residual / softmax).
# Measured on one H100 80GB HBM3 (400 W): tiny tower <= 5.1e-4, ViT-H/14 <= 7.5e-4; the bars are twice that.
TOL_TOWER_TINY = 1e-3
TOL_TOWER_FULL = 1.5e-3
TOL_CONCAT = 5e-3          # the VAE encoder's bar (tests/test_pipeline_gpu.py)


def relerr(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm()).item()


def per_frame_relerr(a, b):
    a, b = a.float().cpu().flatten(1), b.float().cpu().flatten(1)
    return ((a - b).norm(dim=1) / b.norm(dim=1)).max().item()


def frames(n, H, W, seed):                      # = oracle/pin_clip.py `frames` / `frame_seed`
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, H, W, generator=g) * 2 - 1


def frame_seed(n, H, W):
    return 1000 + n * 7 + H * 3 + W


@pytest.fixture(scope="module")
def ops():
    from gcd_b200 import ops as o
    o.lib()
    return o


def unpatch(patches, n, stride):
    """[n*257, 640] patch matrix -> the normalised [n, 3, 224, 224] image, subsampled [..., ::stride, ::stride]."""
    p = patches.float().cpu().view(n, 257, 640)[:, 1:, :588].reshape(n, 16, 16, 14, 14, 3)
    img = p.permute(0, 5, 1, 3, 2, 4).reshape(n, 3, 224, 224)
    return img[:, :, ::stride, ::stride]


@pytest.mark.parametrize("n,H,W", [(2, 224, 224), (2, 256, 384), (2, 576, 1024)])
def test_preprocess_vs_golden(ops, n, H, W):
    from gcd_b200 import clip
    gold = torch.load(os.path.join(GOLD, "clip_tiny.pt"))
    x = frames(n, H, W, frame_seed(n, H, W)).cuda()
    eng = clip.ClipEngine.__new__(clip.ClipEngine)                 # the preprocessing needs no weights
    eng.device, eng._taps = x.device, {}
    taps = eng.taps(H, W)
    out = torch.empty(n * 257, 640, device="cuda", dtype=torch.float32)
    scratch = torch.empty(2 * x.numel(), device="cuda") if taps else None
    ms = torch.tensor(clip.OPENAI_MEAN + clip.OPENAI_STD, device="cuda")
    ops.clip_preprocess(x, taps[0] if taps else None, taps[1] if taps else None, ms, out, scratch)
    o = out.view(n, 257, 640).cpu()
    assert torch.all(o[:, 0] == 0) and torch.all(o[:, :, 588:] == 0)
    img = unpatch(out, n, gold["pre_stride"])
    ref = gold[f"pre_{n}x{H}x{W}"]
    e = (img - ref).abs().max().item()
    print(f"preprocess {n}x{H}x{W}: max abs {e:.2e}")
    assert e <= 1e-5
    if (H, W) == (224, 224):                                        # pass-through: the input itself, normalised
        raw = (((x.cpu() + 1) / 2) - torch.tensor(clip.OPENAI_MEAN).view(1, 3, 1, 1)) / torch.tensor(clip.OPENAI_STD).view(1, 3, 1, 1)
        assert (unpatch(out, n, 1) - raw).abs().max().item() <= 1e-6


def _attn_ref(qkv, n, L, heads):
    q, k, v = qkv.float().view(n, L, 3, heads, 80).permute(2, 0, 3, 1, 4)
    o = F.scaled_dot_product_attention(q, k, v)                     # fp32, scale 1/sqrt(80)
    return o.permute(0, 2, 1, 3).reshape(n * L, heads * 80)


@pytest.mark.parametrize("n,L,heads,scale", [(3, 257, 16, 1.0), (2, 129, 16, 1.0), (2, 257, 4, 1.0), (1, 1024, 2, 1.0),
                                             (2, 257, 16, "logit100")])
def test_attention_d80_vs_sdpa(ops, n, L, heads, scale):
    AD = ops.act_dtype()
    g = torch.Generator().manual_seed(L + heads)
    qkv = torch.randn(n * L, 3 * heads * 80, generator=g)
    if scale == "logit100":         # |q.k| / sqrt(80) up to ~100: a near one-hot softmax
        qkv[:, : 2 * heads * 80] *= (100.0 * 80 ** 0.5 / 80) ** 0.5 * 1.2
    qkv = qkv.to(AD).cuda()
    out = torch.empty(n * L, heads * 80, device="cuda", dtype=AD)
    ops.attention_d80(qkv, n, L, heads, out)
    ref = _attn_ref(qkv, n, L, heads)
    if scale == "logit100":
        q, k, _ = qkv.float().view(n, L, 3, heads, 80).permute(2, 0, 3, 1, 4)
        mx = ((q @ k.transpose(-1, -2)) / 80 ** 0.5).abs().max().item()
        assert mx > 60, mx
    e = relerr(out, ref)
    print(f"attention_d80 n={n} L={L} heads={heads} {scale}: rel-L2 {e:.2e}")
    assert e < 2e-3


def test_gelu_epilogue(ops):
    AD = ops.act_dtype()
    M, K, N = 514, 320, 1280
    g = torch.Generator().manual_seed(5)
    x, w = torch.randn(M, K, generator=g).to(AD).cuda(), (torch.randn(N, K, generator=g) * K ** -0.5 * 3).to(AD).cuda()
    b = torch.randn(N, generator=g).cuda()
    ref = F.gelu(x.float() @ w.float().t() + b)
    out32 = torch.empty(M, N, device="cuda")
    ops.linear(x, w, ops.make_ep(out32, bias=b, act=2))
    assert relerr(out32, ref) < 2e-5
    out16 = torch.empty(M, N, device="cuda", dtype=AD)
    ops.linear(x, w, ops.make_ep(out16, bias=b, act=2))
    assert relerr(out16, ref) < 1e-3
    # act 0 / 1 unchanged
    ops.linear(x, w, ops.make_ep(out32, bias=b, act=1))
    assert relerr(out32, F.silu(x.float() @ w.float().t() + b)) < 2e-5


def test_layernorm_f32_with_position_add(ops):
    rows, C = 3 * 257, 1280
    g = torch.Generator().manual_seed(9)
    x, add = torch.randn(rows, C, generator=g).cuda(), torch.randn(257, C, generator=g).cuda()
    gam, bet = (1 + 0.1 * torch.randn(C, generator=g)).cuda(), (0.1 * torch.randn(C, generator=g)).cuda()
    out = torch.empty(rows, C, device="cuda")
    ops.layernorm_f32(x, gam, bet, out, add=add, add_rows_per=1, add_mod=257)
    ref = F.layer_norm(x + add.repeat(3, 1), (C,), gam, bet)
    assert relerr(out, ref) < 1e-6


def _tower(tag):
    from gcd_b200 import synthetic
    from gcd_b200.clip import visual_param_shapes
    from gcd_b200.embedders import FrozenOpenCLIPImageEmbedder
    gold = torch.load(os.path.join(GOLD, f"clip_{tag}.pt"))
    cfg = gold["cfg"]
    emb = FrozenOpenCLIPImageEmbedder(vit_cfg=None if tag == "full" else cfg)
    sd = {"model.visual." + k: v for k, v in synthetic.seeded_state(visual_param_shapes(cfg), seed=0).items()}
    missing, unexpected = emb.load_state_dict(sd, strict=False)
    assert not unexpected and all(not k.startswith("model.visual.") for k in missing)
    return gold, emb.cuda()


@pytest.mark.parametrize("tag", ["tiny", "full"])
def test_tower_vs_golden(tag):
    if not os.path.exists(os.path.join(GOLD, f"clip_{tag}.pt")):
        pytest.skip("golden not generated")
    gold, emb = _tower(tag)
    tol = TOL_TOWER_FULL if tag == "full" else TOL_TOWER_TINY
    for n, H, W in gold["sizes"]:
        z = emb(frames(n, H, W, frame_seed(n, H, W)).cuda())
        ref = gold[f"z_{n}x{H}x{W}"]
        assert z.shape == ref.shape and z.dtype == torch.float32
        e = per_frame_relerr(z, ref)
        print(f"clip[{tag}] {n}x{H}x{W}: max per-frame rel-L2 {e:.2e}")
        assert e < tol


def _hot_path(tag):
    from gcd_b200 import spec, synthetic
    from gcd_b200.pipeline import GCDHotPath
    gold = torch.load(os.path.join(GOLD, f"cond_{tag}.pt"))
    ucfg = spec.UNET_TINY if "kubric" in tag else dict(spec.UNET_TINY, aux_emb_dim=0)
    pipe = GCDHotPath(ucfg, spec.VAE_TINY, num_steps=2, num_frames=14, device="cuda")
    from gcd_b200.clip import visual_param_shapes
    vst = synthetic.seeded_state(visual_param_shapes(gold["vit_cfg"]), seed=gold["vit_seed"])
    pipe.load_clip({"model.visual." + k: v for k, v in vst.items()}, vit_cfg=gold["vit_cfg"])
    pipe.load_cond_encoder(synthetic.seeded_state(spec.encoder_param_shapes(gold["enc_cfg"]), seed=gold["enc_seed"]),
                           gold["quant_w"], gold["quant_b"], enc_cfg=gold["enc_cfg"])
    if "kubric" in tag:
        pipe.load_spherical(gold["sph_w"], gold["sph_b"])
    return gold, pipe, ucfg


@pytest.mark.parametrize("tag", ["kubric_tiny", "pardom_tiny"])
def test_condition_vs_golden(tag):
    gold, pipe, _ = _hot_path(tag)
    c, uc = pipe.condition(gold["batch"])
    for d, ref in ((c, gold["c"]), (uc, gold["uc"])):
        assert set(d) == set(ref)
        for k in ref:
            assert d[k].shape == ref[k].shape and d[k].dtype == ref[k].dtype, k
        # the timestep / spherical embedding kernels' own bars (tests/test_ops_gpu.py): device cosf / sinf vs the host libm
        assert (d["vector"].cpu() - ref["vector"]).abs().max().item() < 2e-5 * max(1.0, ref["vector"].abs().max().item())
    assert torch.equal(uc["vector"], c["vector"])
    assert torch.count_nonzero(uc["crossattn"]) == 0 and torch.count_nonzero(uc["concat"]) == 0
    e_ca, e_cc = per_frame_relerr(c["crossattn"], gold["c"]["crossattn"]), relerr(c["concat"], gold["c"]["concat"])
    print(f"condition[{tag}]: crossattn per-frame rel-L2 {e_ca:.2e}, concat rel-L2 {e_cc:.2e}")
    assert e_ca < TOL_TOWER_TINY and e_cc < TOL_CONCAT


def test_condition_then_sample_video_takes_the_fused_path():
    """Input frames + camera angles -> (c, uc) -> sample_video at 14 x 32 x 48 latents, all on this package's kernels."""
    import sys
    from gcd_b200 import spec, synthetic
    gold, pipe, ucfg = _hot_path("kubric_tiny")
    T, H, W = 14, 256, 384
    g = torch.Generator().manual_seed(11)
    vid = torch.rand(T, 3, H, W, generator=g) * 2 - 1
    batch = {"cond_frames_without_noise": vid, "cond_frames": vid + 0.02 * torch.randn(vid.shape, generator=g),
             "fps_id": torch.full((T,), 6.0), "motion_bucket_id": torch.full((T,), 127.0), "cond_aug": torch.full((T,), 0.02),
             "scaled_relative_angles": torch.tensor([[0.5, -0.1, 1.0]]).repeat(T, 1)}
    c, uc = pipe.condition(batch)
    assert c["concat"].shape == (T, 4, 32, 48) and c["crossattn"].shape == (T, 1, ucfg["context_dim"])
    pipe.load_state(synthetic.seeded_state(spec.unet_param_shapes(ucfg), seed=0),
                    synthetic.seeded_state(spec.decoder_param_shapes(spec.VAE_TINY), seed=0))
    z, out = pipe.sample_video(torch.randn(T, 4, 32, 48, generator=g), c, uc)
    assert pipe.sampler.last_path == "fused"
    assert out.shape == (T, 3, H, W) and torch.isfinite(out).all()
    assert "open_clip" not in sys.modules and "kornia" not in sys.modules
