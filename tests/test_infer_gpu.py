"""gcd_b200.infer on the device: gcd_frames_prepare against the float64 frame oracle (oracle/frames_oracle.py), and the command
line end to end on a PNG folder, a single image and an mp4 (when cv2 imports) with the tiny seeded model and a checkpoint written as
tests/test_evaluate_gpu.py writes one.

Tolerance. The kernel takes the two weighted sums of the resize as unfused fp32 roundings, the oracle in float64 rounded once:
they differ by at most two fp32 ulps at 1.0 (2.4e-7). Without a resize the value is u8 / 255 and the round trip in fp32 on
both sides: equal."""
import importlib.util
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu
TOL = 2.4e-7
T, S, STEPS, FRAME_HW = 14, 2, 2, (64, 128)


def _prepare(u8, frame_hw, center_crop=True, channel_map=(0, 1, 2)):
    from gcd_b200 import infer as I, ops
    from oracle import frames_oracle as F
    n, H, W, _ = u8.shape
    out = torch.full((n, 3, *frame_hw), float("nan"), device="cuda")
    ops.frames_prepare(torch.from_numpy(u8).cuda(), I.crop_box(H, W, frame_hw, center_crop), out, channel_map)
    want = torch.from_numpy(F.prepare(u8, frame_hw, center_crop, channel_map))
    return out.cpu(), want


CASES = (  # (label, n, H, W, C, frame_hw, center_crop, channel_map, exact)
    ("no-op", 2, 64, 96, 3, (64, 96), True, (0, 1, 2), True),
    ("crop only", 2, 64, 100, 3, (64, 96), True, (0, 1, 2), True),
    ("exact 2x down", 2, 128, 192, 3, (64, 96), True, (0, 1, 2), False),
    ("426x640 -> 256x384", 2, 426, 640, 3, (256, 384), True, (0, 1, 2), False),
    ("upscale", 2, 48, 80, 3, (64, 128), True, (0, 1, 2), False),
    ("no crop, stretch", 1, 50, 70, 3, (64, 128), False, (0, 1, 2), False),
    ("RGBA", 2, 90, 120, 4, (64, 128), True, (0, 1, 2), False),
    ("BGR", 2, 1080, 1920, 3, (256, 384), True, (2, 1, 0), False),
)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_frames_prepare_matches_oracle(case):
    label, n, H, W, C, hw, cc, cmap, exact = case
    u8 = np.random.default_rng(n * H + W).integers(0, 256, (n, H, W, C), dtype=np.uint8)
    got, want = _prepare(u8, hw, cc, cmap)
    assert torch.isfinite(got).all() and 0 <= got.min() and got.max() <= 1
    err = (got.double() - want.double()).abs().max().item()
    print(f"{label}: max |kernel - oracle| {err:.2e}, equal {(got == want).double().mean().item():.3f}")
    if exact:
        assert torch.equal(got, want), label
    assert err <= TOL, label


def test_prepare_frames_groups_mixed_sizes_and_stills():
    from gcd_b200 import infer as I
    from oracle import frames_oracle as F
    rng = np.random.default_rng(9)
    a, b = (torch.from_numpy(rng.integers(0, 256, s, dtype=np.uint8)) for s in ((70, 100, 3), (64, 128, 4)))
    images = [a, b, a.clone(), b, b]                  # b three times as one tensor: a still, prepared once
    got = I.prepare_frames(images, FRAME_HW, True, (0, 1, 2), "cuda").cpu()
    for i, img in enumerate(images):
        want = torch.from_numpy(F.prepare(img.numpy()[None], FRAME_HW))[0]
        assert (got[i].double() - want.double()).abs().max().item() <= TOL, i


def _evaluate_test_module():
    spec = importlib.util.spec_from_file_location("_evaluate_gpu_helpers", os.path.join(ROOT, "tests", "test_evaluate_gpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    from torchvision.io import write_png
    root = tmp_path_factory.mktemp("infer")
    ck = str(root / "kubric_gradual_max90.ckpt")
    gold = _evaluate_test_module()._write_checkpoint(ck)
    mc = root / "model.json"
    mc.write_text(json.dumps({"unet": {"model_channels": 64}, "vae": {"ch": 64}, "encoder": gold["enc_cfg"], "vit": gold["vit_cfg"]}))
    rng = np.random.default_rng(4)
    folder = root / "my_frames"
    folder.mkdir()
    for t in range(T + 2):
        write_png(torch.from_numpy(rng.integers(0, 256, (3, 48, 100), dtype=np.uint8)), str(folder / f"{t:04d}.png"))
    still = root / "still_rgb.png"
    from PIL import Image                             # torchvision writes no RGBA PNG
    Image.fromarray(rng.integers(0, 256, (70, 120, 4), dtype=np.uint8), "RGBA").save(str(still))
    examples = [str(folder), str(still)]
    try:
        import cv2
        mp4 = str(root / "clip.mp4")
        w = cv2.VideoWriter(mp4, cv2.VideoWriter_fourcc(*"mp4v"), 12.0, (160, 72))
        for t in range(2 * T):
            w.write(rng.integers(0, 256, (72, 160, 3), dtype=np.uint8))
        w.release()
        examples.append(mp4)
    except ImportError:
        cv2 = None
    return dict(root=root, ck=ck, mc=str(mc), examples=examples, mp4=cv2 is not None)


def _argv(inputs, out, num_samples=S, extra=()):
    return ["--kind", "kubric", "--checkpoint", inputs["ck"], "--model-config", inputs["mc"], "--input", *inputs["examples"],
            "--output", str(out), "--num-samples", str(num_samples), "--num-steps", str(STEPS), "--frame-height",
            str(FRAME_HW[0]), "--frame-width", str(FRAME_HW[1]), "--frame-stride", "1", "--save-mp4", str(int(inputs["mp4"])),
            "--seed", "3", *extra]


def _png(path):
    from torchvision.io import decode_png, read_file
    return decode_png(read_file(str(path)))


@pytest.fixture(scope="module")
def run(inputs):
    from gcd_b200 import infer as I
    out = inputs["root"] / "a" / "demo_run"
    res = I.main(_argv(inputs, out))
    return dict(out=out, res=res)


def test_outputs_exist_with_frame_counts_and_shapes(inputs, run):
    from gcd_b200 import infer as I
    out, res = run["out"], run["res"]
    assert [r["index"] for r in res] == list(range(len(inputs["examples"])))
    assert json.loads((out / "args_infer.json").read_text())["num_samples"] == S
    names = ["my_frames", "still", "clip"][:len(inputs["examples"])]
    for r, name in zip(res, names):
        stem = r["output"]
        assert stem == os.path.join(str(out), "extra", f"demo_{r['index']:03d}_nkb_gr_m90_{name}")
        for suffix, c in [("_input", 3)] + [(f"_pred_s{s}", 3) for s in range(S)] + [("_uncert", 1)]:
            pngs = sorted(os.listdir(stem + suffix))
            assert pngs == [f"{t:04d}.png" for t in range(T)], suffix
            assert tuple(_png(os.path.join(stem + suffix, pngs[0])).shape) == (c, *FRAME_HW)
            if inputs["mp4"]:
                import cv2
                cap = cv2.VideoCapture(stem + suffix + ".mp4")
                assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == T and cap.get(cv2.CAP_PROP_FPS) == (6 + 12) // 2
                cap.release()
        m = json.loads(open(stem + "_metrics.json").read())
        assert list(m) == ["frame_diversity", "mean_diversity"] and len(m["frame_diversity"]) == T
    still = sorted(os.listdir(res[1]["output"] + "_input"))
    first = _png(os.path.join(res[1]["output"] + "_input", still[0]))
    assert all(torch.equal(first, _png(os.path.join(res[1]["output"] + "_input", p))) for p in still)


def test_predictions_equal_sample_example_and_diversity_matches_float64(inputs, run):
    from gcd_b200 import evaluate as E, infer as I
    args = I.parser().parse_args(_argv(inputs, run["out"]))
    hot, _ = E.load_hotpath(args, "cuda")
    for r in run["res"]:
        g = I.example_generator(args.seed, r["index"], "cuda")
        input_rgb, batch = I.prepare_input(args, r["example"], g, "cuda")
        _, sampled = E.sample_example(hot, batch, S, g, args.decoding_t)
        assert torch.equal(I.quantize(input_rgb).cpu(), torch.stack([_png(os.path.join(r["output"] + "_input", f"{t:04d}.png"))
                                                                     for t in range(T)]))
        for s in range(S):
            want = I.quantize(sampled[s]).cpu()
            got = torch.stack([_png(os.path.join(r["output"] + f"_pred_s{s}", f"{t:04d}.png")) for t in range(T)])
            print(f"{r['example']} sample {s}: {(got != want).sum().item()} differing bytes")
            assert torch.equal(got, want)
        x = sampled.double()
        md = x.std(dim=0, unbiased=False).mean(dim=1).mean(dim=(1, 2)).mean().item()
        got_md = json.loads(open(r["output"] + "_metrics.json").read())["mean_diversity"]
        print(f"mean_diversity {got_md:.6f}, float64 {md:.6f}")
        assert abs(got_md - md) < 1e-6 and md > 0


def test_one_sample_has_zero_diversity(inputs, tmp_path):
    from gcd_b200 import infer as I
    res = I.main(_argv(dict(inputs, examples=inputs["examples"][:1]), tmp_path / "one_run", 1, ["--save-images", "0",
                                                                                               "--save-mp4", "0"]))
    m = json.loads(open(res[0]["output"] + "_metrics.json").read())
    assert m["mean_diversity"] == 0.0 and all(v == 0.0 for v in m["frame_diversity"])
    assert not os.path.exists(res[0]["output"] + "_pred_s0")


def test_two_runs_with_one_seed_write_identical_bytes(inputs, run):
    from gcd_b200 import infer as I
    out2 = inputs["root"] / "b" / "demo_run"
    I.main(_argv(inputs, out2))
    a, b = run["out"] / "extra", out2 / "extra"
    files = sorted(str(p.relative_to(a)) for p in a.rglob("*") if p.is_file())
    assert files == sorted(str(p.relative_to(b)) for p in b.rglob("*") if p.is_file())
    assert any(f.endswith(".png") for f in files) and any(f.endswith("_metrics.json") for f in files)
    differ = [f for f in files if (a / f).read_bytes() != (b / f).read_bytes()]
    assert not differ, differ[:10]
