"""Writes tests/golden/infer_frames.pt and tests/golden/infer_host.pt from the reference's own infer.py path (needs a reference
checkout: GCD_REFERENCE, see oracle/ref_shim.py, and OpenCV).

    python -m oracle.pin_infer

Cut out of the reference sources with `ast` (oracle/pin_evaluate.py's `_cut`) and run unedited on CPU:
  sgm/data/common.py      center_crop_numpy, process_image, load_video_mp4 (with a stub `mediapy.read_video` that returns the given
                          uint8 frames: the fixture starts at decoded frames), construct_trajectory;
  scripts/eval_utils.py   construct_batch, get_list_of_input_images_or_videos, is_image_folder, is_image_file, is_video_file;
  scripts/infer.py        calculate_metrics, process_example (with stubs for everything but the output naming: the stub
                          save_results records the path prefix), and the model-name statement of eval_utils.load_model_bundle.
cv2.resize runs with IPP off (cv2.ipp.setUseIPP(False)): OpenCV's generic INTER_LINEAR path, which the device kernel follows; IPP
builds differ from it by up to 4e-5 at some ratios (426x640 -> 256x384). Inputs are regenerated from seeds or stored when tiny;
only the reference's outputs are stored.
"""
import ast
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from oracle.pin_evaluate import _cut  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
T = 14
# process_image cases: (input H, W, C, output h, w, center_crop, seed); at most 64 x 96 except one 256 x 384 input (exact 2x)
IMAGE_CASES = ((48, 80, 3, 64, 96, 1, 1),      # crop width to 72, upscale
               (64, 96, 4, 64, 96, 1, 2),      # RGBA, no crop, no resize
               (64, 100, 3, 64, 96, 1, 3),     # crop only
               (60, 96, 3, 64, 96, 1, 4),      # crop width to 90, upscale
               (64, 90, 3, 64, 128, 1, 5),     # crop height to 45 (aspect 2), downscale
               (50, 70, 3, 32, 64, 0, 6),      # no crop: stretch
               (256, 384, 3, 128, 192, 1, 7))  # exact 2x down (cv2's INTER_AREA fast path)
# load_video_mp4 cases: (frames N, H, W, clip frames, output h, w, center_crop, seed)
VIDEO_CASES = ((6, 40, 64, (1, 3, 5), 64, 96, 1, 11), (4, 32, 48, (0, 1, 2, 3), 32, 64, 1, 12))
# crop-box cases (H, W, h, w): both crop directions and aspect ratios at the 2e-3 tolerance edge (W / H = 1.5 +- 2e-3 and just past)
CROP_CASES = ((1000, 1502, 256, 384), (1000, 1503, 256, 384), (1000, 1498, 256, 384), (1000, 1497, 256, 384),
              (1080, 1920, 256, 384), (720, 1280, 256, 384), (480, 640, 256, 384), (426, 640, 256, 384), (256, 384, 256, 384),
              (1920, 1080, 256, 384), (333, 500, 64, 128), (100, 99, 64, 64), (101, 100, 64, 64))
# construct_batch model bundles: (label, delta az range, delta el range, trajectory, move_time, camera_control, motion range)
BUNDLES = (("kubric_gradual_max180", [-180.0, 180.0], [-60.0, 60.0], "interpol_linear", 13, "spherical", [0, 255]),
           ("kubric_gradual_max90", [-90.0, 90.0], [-30.0, 30.0], "interpol_linear", 13, "spherical", [0, 255]),
           ("kubric_direct_max90", [-90.0, 90.0], [-30.0, 30.0], "interpol_linear", 0, "spherical", [0, 255]),
           ("kubric_sine", [-90.0, 90.0], [-30.0, 30.0], "interpol_sine", 7, "spherical", [0, 255]),
           ("pardom_gradual", [0.0, 0.0], [0.0, 0.0], "interpol_linear", 0, "none", [127, 127]))
# (delta azimuth, elevation, radius, frame_rate, motion_id, cond_aug, force_custom_mbid)
CONTROLS = ((30.0, 15.0, 0.0, 12, 127, 0.02, 0), (-75.5, 5.0, 1.5, 8, 127, 0.02, 0), (30.0, 15.0, 0.0, 12, 40, 0.05, 1))
# input tree of the discovery fixture: files created empty, then the paths given to the reference
TREE = ("vids/a.mp4", "vids/b.MOV", "vids/notes.md", "frames1/0000.png", "frames1/0001.png", "frames1/0002.jpg",
        "frames1/readme.txt", "half/0.png", "half/x.txt", "nested/s1/0.png", "nested/s1/1.png", "nested/s2/clip.mp4",
        "single.jpg")
LIST_TXT = "# a comment\n\n  vids/a.mp4  \nsome/other_clip.mp4\n#frames1\nframes1\n"
DISCOVERY = (["vids/a.mp4"], ["frames1"], ["nested"], ["list.txt"], ["single.jpg"], ["vids/*.mp4"], ["."],
             ["half", "single.jpg", "missing/*.png"])
# (output directory, example index, example, checkpoint)
NAMES = (("out/demo_run", 0, "clips/my_video.mp4", "pretrained/kubric_gradual_max90.ckpt"),
         ("out/dbg1", 7, "frames/scene_p0_rgb", "pretrained/pardom_direct_semantic.ckpt"),
         ("/abs/test", 12, "img/photo.jpeg", "logs/2024_run_abc/checkpoints/last.ckpt"))


def seeded_frames(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, size=shape, dtype=np.uint8)


def seeded_samples(seed=21, S=3, H=8, W=12):
    return torch.rand(S, T, 3, H, W, generator=torch.Generator().manual_seed(seed))


def seeded_input(seed):
    return torch.rand(T, 3, 4, 6, generator=torch.Generator().manual_seed(seed))


def make_tree(root):
    for p in TREE:
        path = os.path.join(root, p)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        open(path, "w").close()
    with open(os.path.join(root, "list.txt"), "w") as f:
        f.write(LIST_TXT)


def reference():
    import cv2
    from einops import rearrange
    if not ref_shim.available():
        raise RuntimeError("set GCD_REFERENCE to the gcd-model directory of a basilevh/gcd checkout")
    noprint = lambda *a, **k: None
    common_py = os.path.join(ref_shim.REF, "sgm", "data", "common.py")
    eval_py = os.path.join(ref_shim.REF, "scripts", "eval_utils.py")
    infer_py = os.path.join(ref_shim.REF, "scripts", "infer.py")
    video = {}
    mediapy = types.SimpleNamespace(read_video=lambda fp: video[fp])
    ns = dict(np=np, cv2=cv2, os=os, rearrange=rearrange, mediapy=mediapy, print=noprint)
    exec(compile(_cut(common_py, ["center_crop_numpy", "process_image", "load_video_mp4", "construct_trajectory"]), common_py,
                 "exec"), ns)
    common = types.SimpleNamespace(construct_trajectory=ns["construct_trajectory"])
    ens = dict(np=np, os=os, glob=__import__("glob"), common=common, print=noprint,
               image_extensions=[".jpg", ".jpeg", ".png", ".bmp", ".tiff"],
               video_extensions=[".mp4", ".avi", ".mov", ".flv", ".mkv", ".webm"])
    exec(compile(_cut(eval_py, ["construct_batch", "get_list_of_input_images_or_videos", "is_image_folder", "is_image_file",
                                "is_video_file"]), eval_py, "exec"), ens)
    # the model-name statement of load_model_bundle
    src = open(eval_py).read()
    fn = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "load_model_bundle")
    stmt = next(n for n in fn.body if isinstance(n, ast.If) and "/checkpoints" in ast.get_source_segment(src, n.test))
    name_code = compile(ast.Module(body=[stmt], type_ignores=[]), eval_py, "exec")

    def model_name(model_path):
        loc = dict(model_path=model_path, os=os)
        exec(name_code, loc)
        return loc["model_name"]

    saved = []
    ins = dict(np=np, os=os, time=__import__("time"), print=noprint,
               load_input=lambda *a: (None, np.zeros(6, np.float32), None), run_inference=lambda *a: [],
               calculate_metrics=lambda *a: ({}, None), get_controls_friendly=lambda c: (False, "", "fs0_fr0"),
               create_visualizations=lambda *a: {}, save_results=lambda *a: saved.append(a[-1]))
    exec(compile(_cut(infer_py, ["calculate_metrics", "process_example"]), infer_py, "exec"), ins)
    calc = ins["calculate_metrics"]
    ins["calculate_metrics"] = lambda *a: ({}, None)

    def output_prefix(output, index, example, model):
        args = types.SimpleNamespace(output=output, num_samples=0)
        ins["process_example"](args, 0, index, example, [None, None, None, "cpu", model])
        return saved.pop()

    return dict(ns=ns, eval=ens, video=video, model_name=model_name, output_prefix=output_prefix, calculate_metrics=calc)


def main():
    import cv2
    cv2.ipp.setUseIPP(False)
    ref = reference()
    ns, ens = ref["ns"], ref["eval"]

    crops = []
    for H, W, h, w in CROP_CASES:
        yx = np.stack(np.meshgrid(np.arange(H), np.arange(W), indexing="ij"), -1)
        c = ns["center_crop_numpy"](yx, w / h, False)
        crops.append(dict(H=H, W=W, frame_hw=(h, w), box=(int(c[0, 0, 0]), int(c[0, 0, 1]), c.shape[0], c.shape[1])))

    images = []
    for H, W, C, h, w, cc, seed in IMAGE_CASES:
        u8 = seeded_frames((H, W, C), seed)
        out = ns["process_image"](u8, cc, w, h, False)                      # [3, h, w] in [-1, 1]
        images.append(dict(shape=(H, W, C), frame_hw=(h, w), center_crop=cc, seed=seed,
                           input_rgb=torch.from_numpy((out + 1.0) / 2.0)))    # infer.py:137
    videos = []
    for N, H, W, frames, h, w, cc, seed in VIDEO_CASES:
        u8 = seeded_frames((N, H, W, 3), seed)
        ref["video"]["clip.mp4"] = u8
        out = ns["load_video_mp4"]("clip.mp4", np.array(frames), cc, w, h, False)
        videos.append(dict(shape=(N, H, W, 3), frames=frames, frame_hw=(h, w), center_crop=cc, seed=seed,
                           input_rgb=torch.from_numpy((out + 1.0) / 2.0)))
    torch.save(dict(crops=crops, images=images, videos=videos,
                    meta={"source": "gcd-model/sgm/data/common.py center_crop_numpy / process_image / load_video_mp4, cut with "
                                    "ast and run unedited; cv2 " + cv2.__version__ + " with IPP off"}),
               os.path.join(GOLD, "infer_frames.pt"))

    batches = []
    for bi, (label, az, el, traj, mt, cam, mbr) in enumerate(BUNDLES):
        bundle = [None, None, None, "cpu", label, az, el, [0.0, 0.0], traj, mt, cam, mbr]
        for ci, (da, de, dr, fr, mid, ca, force) in enumerate(CONTROLS):
            controls = np.array([0, 2, fr, da, de, dr], dtype=np.float32)
            seed = 1000 + 10 * bi + ci
            x = seeded_input(seed).numpy()
            torch.manual_seed(seed)
            b = ens["construct_batch"](x, controls[3], controls[4], controls[5], T, controls[2], mid, ca, force, bundle, "cpu")
            batches.append(dict(bundle=bi, controls=ci, seed=seed, batch=b))
    with tempfile.TemporaryDirectory() as tmp:
        make_tree(tmp)
        cwd = os.getcwd()
        os.chdir(tmp)
        try:
            discovery = [(paths, ens["get_list_of_input_images_or_videos"](paths)) for paths in DISCOVERY]
        finally:
            os.chdir(cwd)
    names = [(o, i, e, c, ref["model_name"](c), ref["output_prefix"](o, i, e, ref["model_name"](c))) for o, i, e, c in NAMES]
    S = seeded_samples()
    m, unc = ref["calculate_metrics"](None, [dict(sampled_rgb=s.numpy()) for s in S])
    diversity = dict(uncertainty=torch.from_numpy(unc), frame_diversity=torch.from_numpy(m["frame_diversity"]),
                     mean_diversity=float(m["mean_diversity"]))
    torch.save(dict(bundles=BUNDLES, controls=CONTROLS, batches=batches, discovery=discovery, names=names, diversity=diversity,
                    meta={"source": "gcd-model/scripts/eval_utils.py construct_batch / get_list_of_input_images_or_videos, "
                                    "infer.py calculate_metrics / process_example naming, cut with ast and run unedited"}),
               os.path.join(GOLD, "infer_host.pt"))
    for f in ("infer_frames.pt", "infer_host.pt"):
        print(f, os.path.getsize(os.path.join(GOLD, f)))


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
