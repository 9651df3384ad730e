"""fp64 / fp32 torch restatement of the reference's point-cloud view synthesis (TEST INFRASTRUCTURE). Runs on any device, one render
at a time, as the reference does on its data GPU:

    project_points_to_pixels   gcd-model/sgm/data/geometry.py:242-344
    spreaded_index_add         geometry.py:347-401
    blur_into_black            geometry.py:404-424, gaussian_blur_masked_vectorized geometry.py:427-444
    bilinear resize, `* 2 - 1` kubric_arbit.py:463-467 / 551-562, pardom_arbit.py:697-701 / 724-733
    synth_src_dst_rgb          kubric_arbit.py:410-563
    synth_rgb                  pardom_arbit.py:585-738

torchvision's `gaussian_blur` (kernel from linspace / exp / normalise, outer product by mm, 'reflect' padding, depthwise conv2d) is
restated here so the oracle imports nothing beyond torch. Non-finite camera coordinates follow the reference's CPU run: the NaN uv
casts to INT_MIN and the point is dropped."""
import torch
import torch.nn.functional as F


def spread_offsets(radius):
    """spreaded_index_add's neighbour offsets (dx, dy), in the reference's order."""
    left, right = radius // 2, (radius + 1) // 2
    return [(dx, dy) for dx in range(-left, right + 1) for dy in range(-left, right + 1) if (dx, dy) != (0, 0)]


def _index_add_spread(t, inds, vals, H, W, radius):
    t.index_add_(0, inds, vals)
    for dx, dy in spread_offsets(radius):
        x, y = inds % W + dx, inds // W + dy
        m = (x >= 0) & (x < W) & (y >= 0) & (y < H)
        t.index_add_(0, (y * W + x)[m], vals[m] * 0.02)


def project(xyz, col, K, RT, H, W, spread_radius):
    """xyz [N, 3], col [N, 3] (float32 colours in [0, 1]); K, RT camera matrices. Returns float32 [H, W, 3] in [0, 1]."""
    xyz, col = xyz.double(), col.double()
    K, RT = K.double().to(xyz.device), RT.double().to(xyz.device)
    cam = (xyz - RT[0:3, 3]) @ RT[0:3, 0:3]
    uv = torch.mm(K, cam.T).T
    uv = uv[:, 0:2] / uv[:, 2:3]
    a = uv + 0.5
    # (a).type(int32) truncates toward zero; out-of-range and NaN become INT_MIN on CPU (dropped)
    ok = torch.isfinite(a).all(dim=1) & (a[:, 0] > -1) & (a[:, 0] < W) & (a[:, 1] > -1) & (a[:, 1] < H) & (cam[:, 2] > 0.1)
    a, col, depth = a[ok], col[ok], cam[ok][:, 2:3]
    if depth.numel() == 0:
        raise ValueError("no point lands in the image")
    ij = a.trunc().long()
    inds = ij[:, 1] * W + ij[:, 0]
    if depth.max() >= 64.0:
        strength = 256.0
        depth = torch.clamp(torch.sqrt(depth), 0.0, 32.0)
    else:
        strength = 512.0
    dn = depth / depth.max() * 2.0 - 1.0
    w = torch.exp(-dn * strength)
    pw = torch.zeros(H * W, 1, dtype=torch.float64, device=xyz.device)
    _index_add_spread(pw, inds, w, H, W, spread_radius)
    img = torch.zeros(H * W, 3, dtype=torch.float64, device=xyz.device)
    _index_add_spread(img, inds, col * w, H, W, spread_radius)
    pw = pw.view(H, W, 1)
    pw[pw <= 0.0] = -1.0
    return torch.clamp(img.view(H, W, 3) / pw, 0.0, 1.0).to(torch.float32)


def gaussian_kernel1d(k, sigma, dtype, device=None):
    half = (k - 1) * 0.5
    x = torch.linspace(-half, half, steps=k, dtype=dtype, device=device)
    pdf = torch.exp(-0.5 * (x / sigma).pow(2))
    return pdf / pdf.sum()


def gaussian_blur(img, k, sigma):
    """torchvision.transforms.functional.gaussian_blur for a float [C, H, W] tensor: the kernel in the image's dtype."""
    k1 = gaussian_kernel1d(k, sigma, img.dtype, img.device)
    k2 = torch.mm(k1[:, None], k1[None, :])
    C = img.shape[0]
    x = F.pad(img[None], [k // 2] * 4, mode="reflect")
    return F.conv2d(x, k2.expand(C, 1, k, k), groups=C)[0]


def blur_into_black(img, k, sigma):
    """img float32 [H, W, 3] -> float64 [H, W, 3]."""
    black = (img.sum(dim=-1) == 0.0)[None]
    x = img.permute(2, 0, 1)
    borrow = (~black).to(torch.float64)
    leak = gaussian_blur(x, k, sigma) / gaussian_blur(borrow, k, sigma).clamp(min=1e-7)
    x2 = x * (~black) + leak * black
    return gaussian_blur(x2, 3, 0.6).permute(1, 2, 0)


def render(xyz, col, K, RT, render_hw, frame_hw, spread_radius, k):
    """One render through the whole chain: float64 [3, Hp, Wp] in [0, 1] (before `* 2 - 1`)."""
    H, W = render_hw
    img = blur_into_black(project(xyz, col, K, RT, H, W, spread_radius), k, k / 4.0)
    return F.interpolate(img.permute(2, 0, 1)[None], tuple(frame_hw), mode="bilinear", align_corners=False)[0]


def colours(rgb_u8, segm=None, palette=None, alpha=0.0):
    """(u8 / 255.0) in float32, optionally blended with palette[segm] as pardom_arbit.py:644-665 does."""
    c = (rgb_u8 / 255.0).to(torch.float32)
    if segm is None or alpha == 0.0:
        return c
    s = palette.to(c.device)[segm.long().flatten()].reshape(c.shape)
    if alpha == 1.0:
        return s
    return (1.0 - alpha) * c + alpha * s


def pixel_intrinsics(intr, render_hw, old_ar):
    H, W = render_hw
    K = intr.clone().to(torch.float32)
    K[..., 0, :] *= W
    K[..., 1, :] *= H
    new_ar = W / H
    if new_ar > old_ar + 1e-3:
        K[..., 1, 1] = K[..., 0, 0]
    elif new_ar < old_ar - 1e-3:
        K[..., 0, 0] = K[..., 1, 1]
    return K


def kubric_views(pcl_xyz, pcl_rgb, intrinsics0, extrinsics_src, extrinsics_dst, reproject=False, render_hw=(280, 420),
                 frame_hw=(256, 384), spread_radius=1):
    """synth_src_dst_rgb restated; pcl_* [T, V, N, 3]. Returns float32 (rgb_src, rgb_dst, reproject | None) [T, 3, Hp, Wp]."""
    K = pixel_intrinsics(intrinsics0, render_hw, 576.0 / 384.0)
    src, dst, rep = [], [], []
    for t in range(pcl_xyz.shape[0]):
        xyz = pcl_xyz[t].float().reshape(-1, 3)
        col = colours(pcl_rgb[t]).reshape(-1, 3)
        src.append(render(xyz, col, K, extrinsics_src[t], render_hw, frame_hw, spread_radius, 21))
        dst.append(render(xyz, col, K, extrinsics_dst[t], render_hw, frame_hw, spread_radius, 21))
        if reproject:
            rep.append(render(pcl_xyz[t][4].float(), colours(pcl_rgb[t][4]), K, extrinsics_dst[t], render_hw, frame_hw,
                              spread_radius, 3))
    f = lambda L: (torch.stack(L) * 2.0 - 1.0).to(torch.float32)
    return f(src), f(dst), (f(rep) if reproject else None)


def pardom_alpha(t, modal_time):
    if 0 < t < modal_time:
        return t / modal_time
    return 0.0 if (t == 0 and 0 < modal_time) else 1.0


def pardom_views(pcl_xyz, pcl_rgb, intrinsics, extrinsics, modality="rgb", segm=None, palette=None, modal_time=0,
                 reproject=False, render_hw=(280, 420), frame_hw=(256, 384), spread_radius=1):
    """synth_rgb restated; pcl_* [T, V, N, 3], segm [T, V, N, 1]. Returns float32 (rgb, reproject | None) [T, 3, Hp, Wp]."""
    K = pixel_intrinsics(intrinsics, render_hw, 640.0 / 480.0)
    out, rep = [], []
    for t in range(pcl_xyz.shape[0]):
        a = pardom_alpha(t, modal_time) if modality == "segm" else 0.0
        col = colours(pcl_rgb[t], None if segm is None else segm[t], palette, a)      # [V, N, 3]
        xyz = pcl_xyz[t].float()
        out.append(render(xyz.reshape(-1, 3), col.reshape(-1, 3), K[t], extrinsics[t], render_hw, frame_hw, spread_radius, 21))
        if reproject:
            rep.append(render(xyz[16], col[16], K[t], extrinsics[t], render_hw, frame_hw, spread_radius, 3))
    f = lambda L: (torch.stack(L) * 2.0 - 1.0).to(torch.float32)
    return f(out), (f(rep) if reproject else None)


# ---- seeded scene-like clouds: a smooth depth field unprojected from a ring of cameras (data-gen/convert_pcl_*.py) ----

def look_at(pos, target=(0.0, 0.0, 0.0)):
    """Camera-to-world RT [4, 4] float32 with +z forward, +y down (the convention project_points_to_pixels expects)."""
    pos = torch.as_tensor(pos, dtype=torch.float64)
    fwd = torch.as_tensor(target, dtype=torch.float64) - pos
    fwd = fwd / fwd.norm()
    right = torch.linalg.cross(fwd, torch.tensor([0.0, 0.0, 1.0], dtype=torch.float64))
    right = right / right.norm()
    down = torch.linalg.cross(fwd, right)
    RT = torch.eye(4, dtype=torch.float64)
    RT[0:3, 0], RT[0:3, 1], RT[0:3, 2], RT[0:3, 3] = right, down, fwd, pos
    return RT.to(torch.float32)


def ring_camera(azimuth_deg, radius, height):
    a = torch.deg2rad(torch.tensor(float(azimuth_deg), dtype=torch.float64))
    return look_at((radius * torch.cos(a).item(), radius * torch.sin(a).item(), height))


def synthetic_clouds(kind, T, V, h, w, seed):
    """kind "kubric" (depths ~ 6..20) or "pardom" (street-like: far points up to fp16 overflow). Each view is an h x w depth map
    unprojected from a ring camera. Returns dict with xyz fp16 [T, V, N, 3], rgb uint8 [T, V, N, 3], segm uint8 [T, V, N, 1],
    intrinsics float32 [T, 3, 3] (normalised), view_extrinsics float32 [V, 4, 4], palette float32 [256, 3]."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64)
    fw, fh = (576.0, 384.0) if kind == "kubric" else (640.0, 480.0)
    f = 0.9 * fw
    Kp = torch.tensor([[f / fw * w, 0, 0.5 * w], [0, f / fw * w, 0.5 * h], [0, 0, 1]], dtype=torch.float64)
    u = (torch.arange(w, dtype=torch.float64) + 0.5)[None, :].expand(h, w) / w
    v = (torch.arange(h, dtype=torch.float64) + 0.5)[:, None].expand(h, w) / h
    views = [ring_camera(360.0 * i / V + 7.0 * r(1).item(), 12.0 + 4 * r(1).item(), 2.0 + 3 * r(1).item()) for i in range(V)]
    ph = r(V, 6) * 6.283
    xyz, rgb, segm = [], [], []
    for t in range(T):
        fx, fc, fs = [], [], []
        for i in range(V):
            p = ph[i]
            s = 0.15 * t
            d = (1.0 + 0.25 * torch.sin(3 * u + p[0] + s) * torch.cos(2 * v + p[1]) + 0.1 * torch.sin(9 * u * v + p[2]))
            d = d * (10.0 if kind == "kubric" else 30.0)
            if kind == "pardom":
                sky = v < 0.3 + 0.1 * torch.sin(5 * u + p[3])
                d = torch.where(sky, 1e5 * (1 + u), d)             # fp16 overflows to inf on store
            x = (u * w - Kp[0, 2]) * d / Kp[0, 0]
            y = (v * h - Kp[1, 2]) * d / Kp[1, 1]
            cam = torch.stack([x, y, d], -1).reshape(-1, 3)
            RT = views[i].double()
            world = cam @ RT[0:3, 0:3].T + RT[0:3, 3]
            fx.append(world.to(torch.float16))
            col = torch.stack([0.5 + 0.5 * torch.sin(4 * u + p[k] + k + s) * torch.cos(3 * v + p[5 - k]) for k in range(3)], -1)
            fc.append((col.reshape(-1, 3) * 255).round().clamp(0, 255).to(torch.uint8))
            fs.append(((d / d.max()) * 7 + 3 * (u > 0.5)).floor().reshape(-1, 1).clamp(0, 255).to(torch.uint8))
        xyz.append(torch.stack(fx)); rgb.append(torch.stack(fc)); segm.append(torch.stack(fs))
    K = torch.tensor([[f / fw, 0, 0.5], [0, f / fh, 0.5], [0, 0, 1]], dtype=torch.float32)
    intr = K[None].repeat(T, 1, 1)
    intr[:, 0, 0] *= (1 + 0.01 * torch.arange(T, dtype=torch.float32))
    palette = torch.rand(256, 3, generator=g, dtype=torch.float32)
    return dict(xyz=torch.stack(xyz), rgb=torch.stack(rgb), segm=torch.stack(segm), intrinsics=intr,
                view_extrinsics=torch.stack(views), palette=palette)


def trajectory(T, azimuth0, azimuth1, radius, height):
    """Extrinsics [T, 4, 4] float32 of a ring camera moving from azimuth0 to azimuth1."""
    return torch.stack([ring_camera(azimuth0 + (azimuth1 - azimuth0) * t / max(T - 1, 1), radius, height) for t in range(T)])
