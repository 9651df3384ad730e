"""Point-cloud view synthesis of the Kubric-4D and ParDom-4D evaluation clips on the device: the conditioning video (`rgb_src`),
the target video (`rgb_dst`) and the reprojection baseline whose black pixels define the occluded mask of
`metrics.calculate_metrics`. The reference renders them per frame from the stored clouds (gcd-model/sgm/data/kubric_arbit.py:410-563
`synth_src_dst_rgb`, pardom_arbit.py:585-738 `synth_rgb`, built on geometry.py:242-444). Here every frame and every render of an
example go through the same three kernels (csrc/render.cu). Dataset indexing, file loading and trajectory sampling stay with the
caller, which passes the clouds and the camera matrices. No CPU path."""
import torch

from . import ops

KUBRIC_REPROJECT_VIEW = 4      # kubric_arbit.py:527: the stored view the reprojection baseline starts from
PARDOM_REPROJECT_VIEW = 16     # pardom_arbit.py:674: the forward ego view
BLUR, REPROJECT_BLUR = 21, 3   # blur_into_black kernel sizes (sigma = k / 4)


def _render(xyz, rgb, renders, render_hw, frame_hw, spread_radius, segm=None, palette=None):
    """xyz fp16 [F, P, 3], rgb uint8 [F, P, 3] (device); renders: list of (frame, p0, n, K [3,3], RT [4,4], alpha, blur kernel).
    Returns float32 [len(renders), 3, Hp, Wp]; raises ValueError when a render has no valid point."""
    if xyz.dim() != 3 or xyz.shape[2] != 3 or rgb.shape != xyz.shape:
        raise ValueError(f"xyz and rgb must be [T, P, 3] of the same shape, got {tuple(xyz.shape)} and {tuple(rgb.shape)}")
    if (segm is None) != (palette is None):
        raise ValueError("segm and palette go together")
    if segm is not None and (segm.shape != xyz.shape[:2] or tuple(palette.shape) != (256, 3)):
        raise ValueError(f"segm must be [T, P] and palette [256, 3], got {tuple(segm.shape)} and {tuple(palette.shape)}")
    ops._need_cuda(xyz, rgb, segm, palette)
    H, W = render_hw
    Hp, Wp = frame_hw
    dev = xyz.device
    R = len(renders)
    desc = torch.tensor([[f, p0, n, k] for f, p0, n, _, _, _, k in renders], dtype=torch.int32)
    cams = torch.zeros(R, 24, dtype=torch.float64)
    for i, (_, _, _, K, RT, alpha, _) in enumerate(renders):
        K, RT = K.detach().cpu().double(), RT.detach().cpu().double()
        if K.shape != (3, 3) or RT.shape != (4, 4):
            raise ValueError(f"K must be [3, 3] and RT [4, 4] per frame, got {tuple(K.shape)} and {tuple(RT.shape)}")
        cams[i, 0:9] = K.reshape(9)
        cams[i, 9:18] = RT[0:3, 0:3].reshape(9)
        cams[i, 18:21] = RT[0:3, 3]
        cams[i, 21] = float(alpha)
    xyz = xyz.to(torch.float16).contiguous()
    rgb = rgb.contiguous()
    if segm is not None:
        segm = segm.to(torch.uint8).contiguous()
        palette = palette.to(torch.float32).contiguous()
    acc = torch.empty(R, H * W, 4, dtype=torch.float64, device=dev)
    maxd = torch.empty(R, dtype=torch.float64, device=dev)
    out = torch.empty(R, 3, Hp, Wp, dtype=torch.float32, device=dev)
    ops.render_views(xyz, rgb, segm, palette, desc, cams.to(dev), H, W, Hp, Wp, spread_radius, acc, maxd, out)
    empty = (maxd.cpu() <= 0).nonzero().flatten().tolist()
    if empty:
        raise ValueError(f"no point lands in the image of render(s) {empty} (frames {[renders[i][0] for i in empty]})")
    return out


def _frames(t, T, what, shape):
    if tuple(t.shape) == shape:
        t = t.unsqueeze(0).expand(T, *shape)
    if tuple(t.shape) != (T, *shape):
        raise ValueError(f"{what} must be {list(shape)} or [T, {', '.join(map(str, shape))}], got {tuple(t.shape)}")
    return t


def render_views(xyz, rgb, K, RT, render_hw, frame_hw, spread_radius, blur_kernel, segm=None, palette=None, alpha=None):
    """Renders one view per frame of a point cloud, as the reference's per-frame chain project_points_to_pixels ->
    blur_into_black(k, k / 4) -> bilinear resize -> `* 2 - 1`.

    xyz: fp16 [T, P, 3] world coordinates; rgb: uint8 [T, P, 3]; K: [3, 3] or [T, 3, 3] in pixel units of the render size;
    RT: [4, 4] or [T, 4, 4] camera poses as the datasets store them (world_to_camera: (x - RT[:3, 3]) @ RT[:3, :3]); render_hw / frame_hw: (H, W) of the render and of the output;
    segm: optional uint8 [T, P] (or [T, P, 1]) semantic ids, palette: float32 [256, 3], alpha: per-frame blend of the palette colour
    into rgb (float or [T]; 1 = palette only). All tensors on the device.
    Returns float32 [T, 3, Hp, Wp] in [-1, 1]. Raises ValueError if a frame has no point in the image."""
    if xyz.dim() != 3:
        raise ValueError(f"xyz must be [T, P, 3], got {tuple(xyz.shape)}")
    T, P = xyz.shape[:2]
    K = _frames(K, T, "K", (3, 3))
    RT = _frames(RT, T, "RT", (4, 4))
    if segm is not None and segm.dim() == 3:
        segm = segm[..., 0]
    if alpha is None:
        alpha = 1.0
    alpha = torch.as_tensor(alpha, dtype=torch.float64).cpu().expand(T)
    renders = [(t, 0, P, K[t], RT[t], float(alpha[t]) if segm is not None else 0.0, int(blur_kernel)) for t in range(T)]
    return _render(xyz, rgb, renders, render_hw, frame_hw, spread_radius, segm, palette)


def _pixel_intrinsics(intr, render_hw, old_ar):
    """Normalised intrinsics [..., 3, 3] -> pixel units of the render, with the aspect fix of the synthesizers (float32, as the
    reference computes it on the host: kubric_arbit.py:433-446, pardom_arbit.py:609-621)."""
    H, W = render_hw
    K = intr.detach().cpu().to(torch.float32).clone()
    K[..., 0, :] *= W
    K[..., 1, :] *= H
    new_ar = W / H
    if new_ar > old_ar + 1e-3:
        K[..., 1, 1] = K[..., 0, 0]
    elif new_ar < old_ar - 1e-3:
        K[..., 0, 0] = K[..., 1, 1]
    return K


def _clouds(pcl_xyz, pcl_rgb):
    if pcl_xyz.dim() != 4 or pcl_xyz.shape[-1] != 3 or pcl_rgb.shape != pcl_xyz.shape:
        raise ValueError(f"pcl_xyz and pcl_rgb must be [T, V, N, 3] of the same shape, got {tuple(pcl_xyz.shape)} and "
                         f"{tuple(pcl_rgb.shape)}")
    T, V, N = pcl_xyz.shape[:3]
    return T, V, N, pcl_xyz.reshape(T, V * N, 3), pcl_rgb.reshape(T, V * N, 3)


def kubric_views(pcl_xyz, pcl_rgb, intrinsics0, extrinsics_src, extrinsics_dst, reproject=False, render_hw=(280, 420),
                 frame_hw=(256, 384), spread_radius=1):
    """synth_src_dst_rgb (kubric_arbit.py:410-563) on the device.

    pcl_xyz: fp16 [T, V, N, 3]; pcl_rgb: uint8 [T, V, N, 3]; intrinsics0: [3, 3] normalised to [0, 1]^2 (frame 0's, used for every
    frame); extrinsics_src / extrinsics_dst: [T, 4, 4]. Renders all V views at blur 21 from the source and the destination camera,
    and with `reproject` the stored view 4 alone at blur 3 from the destination camera.
    Returns (rgb_src, rgb_dst, reproject or None), each float32 [T, 3, Hp, Wp] in [-1, 1]."""
    T, V, N, xyz, rgb = _clouds(pcl_xyz, pcl_rgb)
    if reproject and V <= KUBRIC_REPROJECT_VIEW:
        raise ValueError(f"reprojection reads stored view {KUBRIC_REPROJECT_VIEW}; the cloud has {V} views")
    for e, what in ((extrinsics_src, "extrinsics_src"), (extrinsics_dst, "extrinsics_dst")):
        if tuple(e.shape) != (T, 4, 4):
            raise ValueError(f"{what} must be [T, 4, 4] = [{T}, 4, 4], got {tuple(e.shape)}")
    K = _pixel_intrinsics(intrinsics0, render_hw, 576.0 / 384.0)
    if K.shape != (3, 3):
        raise ValueError(f"intrinsics0 must be [3, 3], got {tuple(intrinsics0.shape)}")
    renders = [(t, 0, V * N, K, extrinsics_src[t], 0.0, BLUR) for t in range(T)]
    renders += [(t, 0, V * N, K, extrinsics_dst[t], 0.0, BLUR) for t in range(T)]
    if reproject:
        renders += [(t, KUBRIC_REPROJECT_VIEW * N, N, K, extrinsics_dst[t], 0.0, REPROJECT_BLUR) for t in range(T)]
    out = _render(xyz, rgb, renders, render_hw, frame_hw, spread_radius)
    return out[:T], out[T:2 * T], (out[2 * T:] if reproject else None)


def pardom_alpha(t, modal_time):
    """Palette weight of frame t in the `segm` modality (pardom_arbit.py:644-665): frames before modal_time fade from rgb."""
    if 0 < t < modal_time:
        return t / modal_time
    if t == 0 and 0 < modal_time:
        return 0.0
    return 1.0


def pardom_views(pcl_xyz, pcl_rgb, intrinsics, extrinsics, modality="rgb", segm=None, palette=None, modal_time=0, reproject=False,
                 render_hw=(280, 420), frame_hw=(256, 384), spread_radius=1):
    """synth_rgb (pardom_arbit.py:585-738) on the device.

    pcl_xyz: fp16 [T, V, N, 3] (non-finite far points allowed); pcl_rgb: uint8 [T, V, N, 3]; intrinsics: [T, 3, 3] normalised;
    extrinsics: [T, 4, 4]; modality "rgb" or "segm" (then segm uint8 [T, V, N, 1] or [T, V, N] and palette float32 [256, 3],
    blended in over the first modal_time frames). With `reproject` the stored view 16 alone is rendered at blur 3.
    Returns (rgb, reproject or None), float32 [T, 3, Hp, Wp] in [-1, 1]."""
    T, V, N, xyz, rgb = _clouds(pcl_xyz, pcl_rgb)
    if modality not in ("rgb", "segm"):
        raise ValueError(f"Unknown selected modality: {modality}")
    if reproject and V <= PARDOM_REPROJECT_VIEW:
        raise ValueError(f"reprojection reads stored view {PARDOM_REPROJECT_VIEW}; the cloud has {V} views")
    if tuple(intrinsics.shape) != (T, 3, 3) or tuple(extrinsics.shape) != (T, 4, 4):
        raise ValueError(f"intrinsics must be [T, 3, 3] and extrinsics [T, 4, 4], got {tuple(intrinsics.shape)} and "
                         f"{tuple(extrinsics.shape)}")
    seg = None
    if modality == "segm":
        if segm is None or palette is None:
            raise ValueError("modality 'segm' needs segm and palette")
        seg = segm.reshape(T, V * N)
    K = _pixel_intrinsics(intrinsics, render_hw, 640.0 / 480.0)
    alpha = [pardom_alpha(t, modal_time) if seg is not None else 0.0 for t in range(T)]
    renders = [(t, 0, V * N, K[t], extrinsics[t], alpha[t], BLUR) for t in range(T)]
    if reproject:
        renders += [(t, PARDOM_REPROJECT_VIEW * N, N, K[t], extrinsics[t], alpha[t], REPROJECT_BLUR) for t in range(T)]
    out = _render(xyz, rgb, renders, render_hw, frame_hw, spread_radius, seg, palette if seg is not None else None)
    return out[:T], (out[T:] if reproject else None)
