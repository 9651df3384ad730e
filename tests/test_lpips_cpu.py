"""LPIPS, CPU side: the fp32 oracle (oracle/lpips_oracle.py) against the reference's own outputs (tests/golden/lpips.pt, written by
oracle/pin_lpips.py from the reference's lpips.py run on CPU with seeded weights), the drop-in module's state-dict keys against the
reference's (tests/golden/lpips_keys.json), checkpoint ingest of `lpips.*` keys, and argument checks."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")


def test_oracle_matches_reference_golden_per_layer():
    from oracle import lpips_oracle as O
    g = torch.load(os.path.join(GOLD, "lpips.pt"))
    sd = O.seeded_state(g["meta"]["weight_seed"])
    with torch.no_grad():
        for c, terms, val in zip(g["cases"], g["terms"], g["lpips"]):
            pred, gt = O.pair_inputs(c["n"], c["H"], c["W"], c["seed"])
            t = O.layer_terms(sd, gt, pred)
            assert t.shape == (5, c["n"])
            assert ((t - terms).abs() / terms.abs()).max().item() < 1e-5
            assert ((O.lpips(sd, gt, pred) - val).abs() / val).max().item() < 1e-5
            assert 0.05 < val.min() and val.max() < 0.5                      # a realistic range, not saturated


def test_golden_small_and_odd_sizes():
    g = torch.load(os.path.join(GOLD, "lpips.pt"))
    assert os.path.getsize(os.path.join(GOLD, "lpips.pt")) < 1 << 20
    assert any(c["H"] % 2 or c["W"] % 2 or (c["H"] // 2) % 2 for c in g["cases"])


def test_module_keys_match_reference():
    from gcd_b200.lpips import LPIPS
    ref = [(k, list(s)) for k, s in json.load(open(os.path.join(GOLD, "lpips_keys.json")))]
    mine = [(k, list(v.shape)) for k, v in LPIPS().state_dict().items()]
    assert sorted(mine) == sorted(ref)
    m = LPIPS()
    assert all(not p.requires_grad for p in m.parameters())
    assert m.scaling_layer.shift.flatten().tolist() == pytest.approx([-0.030, -0.088, -0.188])
    assert m.scaling_layer.scale.flatten().tolist() == pytest.approx([0.458, 0.448, 0.450])


def test_constructor_imports_no_torchvision():
    code = ("import sys; sys.path.insert(0, %r)\n"
            "from gcd_b200.lpips import LPIPS\n"
            "LPIPS()\n"
            "assert 'torchvision' not in sys.modules, 'torchvision imported'\n" % ROOT)
    subprocess.run([sys.executable, "-c", code], check=True, timeout=300)


def test_hotpathroot_loads_lpips_keys(tmp_path):
    from gcd_b200 import checkpoint, spec
    from gcd_b200.lpips import LPIPS
    from gcd_b200.unet import VideoUNet
    from gcd_b200.vae import VideoDecoder
    from oracle import lpips_oracle as O

    def root(**kw):
        return checkpoint.HotPathRoot(VideoUNet(**spec.unet_ctor_kwargs(spec.UNET_TINY)),
                                      VideoDecoder(**spec.decoder_ctor_kwargs(spec.VAE_TINY)), **kw)
    r = root(lpips=LPIPS())
    sd = {k: torch.randn(v.shape) for k, v in r.state_dict().items() if not k.startswith("lpips.")}
    lp = O.seeded_state(3)
    sd.update({"lpips." + k: v for k, v in lp.items()})
    sd["loss.logvar"] = torch.zeros(1)
    path = str(tmp_path / "engine.ckpt")
    torch.save({"state_dict": sd}, path)
    missing, unexpected = r.init_from_ckpt(path)
    assert missing == [] and unexpected == ["loss.logvar"]
    for k, v in lp.items():
        assert torch.equal(r.state_dict()["lpips." + k], v), k
    # without lpips= the module tree is as before: the lpips.* keys stay unexpected
    bare = root()
    assert not any(k.startswith("lpips.") for k in bare.state_dict())
    missing, unexpected = bare.init_from_ckpt(path)
    assert missing == [] and sorted(unexpected) == sorted(["loss.logvar"] + ["lpips." + k for k in lp])


def test_api_rejects_cpu_tensors_and_bad_shapes():
    from gcd_b200 import metrics
    from gcd_b200._lib import GcdError
    from gcd_b200.lpips import LPIPS
    m = LPIPS()
    x = torch.zeros(2, 3, 32, 32)
    with pytest.raises(GcdError):
        m(x, x)                                                   # CPU tensors: there is no CPU path
    with pytest.raises(GcdError):
        metrics.frame_lpips(x, x, m)
    with pytest.raises(ValueError):
        m(x, x[:1])                                               # shapes differ
    with pytest.raises(ValueError):
        m(x[:, :2], x[:, :2])                                     # not RGB
    with pytest.raises(ValueError):
        m(x[..., :8, :8], x[..., :8, :8])                         # too small for relu5_3
    with pytest.raises(ValueError):
        m.layer_distances(torch.zeros(3, 3, 32, 32), x)           # 3 inputs do not pair with 2 targets
    with pytest.raises(ValueError):
        metrics.frame_lpips(torch.zeros(2, 3, 3, 32, 32), torch.zeros(4, 3, 32, 32), m)
