"""Writes tests/golden/lpips.pt and tests/golden/lpips_keys.json from the reference's own LPIPS (needs a reference checkout:
GCD_REFERENCE, see oracle/ref_shim.py) and asserts oracle/lpips_oracle.py against it.

    python -m oracle.pin_lpips

`LPIPS`, `ScalingLayer`, `NetLinLayer`, `vgg16`, `normalize_tensor` and `spatial_average` are cut out of
sgm/modules/autoencoding/lpips/loss/lpips.py with `ast` and run on CPU. Nothing touches the network: `models.vgg16` is
torchvision's constructor with `weights=None`, `load_from_pretrained` is replaced by a no-op before anything is constructed, and
`get_ckpt_path` raises if called. The weights are seeded (lpips_oracle.seeded_state) and loaded with load_state_dict; the inputs are
regenerated from seeds (lpips_oracle.pair_inputs); only the reference's outputs and state-dict keys are stored.
"""
import ast
import json
import os
import sys
import textwrap
import types
from collections import namedtuple

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import lpips_oracle as O  # noqa: E402
from oracle import ref_shim  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
WEIGHT_SEED = 0
# odd sizes exercise floor-mode pooling (50 x 70 -> 25 x 35 -> 12 x 17 -> 6 x 8 -> 3 x 4)
CASES = [dict(n=3, H=64, W=96, seed=1), dict(n=2, H=50, W=70, seed=2)]
NAMES = ("LPIPS", "ScalingLayer", "NetLinLayer", "vgg16", "normalize_tensor", "spatial_average")


def _no_download(*a, **k):
    raise RuntimeError("pin_lpips: the reference tried to fetch LPIPS weights")


def reference():
    """The reference module namespace, executed from its source with the substitutions above."""
    import torchvision
    if not ref_shim.available():
        raise RuntimeError("set GCD_REFERENCE to the gcd-model directory of a basilevh/gcd checkout")
    path = os.path.join(ref_shim.REF, "sgm", "modules", "autoencoding", "lpips", "loss", "lpips.py")
    src = open(path).read()
    body = [n for n in ast.parse(src).body if isinstance(n, (ast.ClassDef, ast.FunctionDef)) and n.name in NAMES]
    assert sorted(n.name for n in body) == sorted(NAMES), [n.name for n in body]
    code = "\n\n".join(textwrap.dedent(ast.get_source_segment(src, n)) for n in body)
    models = types.SimpleNamespace(vgg16=lambda pretrained=True, **kw: torchvision.models.vgg16(weights=None))
    ns = dict(torch=torch, nn=nn, namedtuple=namedtuple, models=models, get_ckpt_path=_no_download)
    exec(compile(code, path, "exec"), ns)
    ns["LPIPS"].load_from_pretrained = lambda self, name="vgg_lpips": None
    return ns


def reference_terms(ns, model, x, y):
    """The reference forward, keeping each layer's term ([5, n]) and the returned value ([n])."""
    outs0, outs1 = model.net(model.scaling_layer(x)), model.net(model.scaling_layer(y))
    lins = [model.lin0, model.lin1, model.lin2, model.lin3, model.lin4]
    terms = [ns["spatial_average"](lins[k].model((ns["normalize_tensor"](outs0[k]) - ns["normalize_tensor"](outs1[k])) ** 2),
                                   keepdim=True) for k in range(5)]
    return torch.stack([t.flatten() for t in terms]), model(x, y).flatten()


def main():
    torch.manual_seed(0)
    ns = reference()
    model = ns["LPIPS"]().eval()
    sd = O.seeded_state(WEIGHT_SEED)
    model.load_state_dict(sd, strict=True)
    keys = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    out = {"meta": {"weight_seed": WEIGHT_SEED, "torch": str(torch.__version__),
                    "source": "sgm/modules/autoencoding/lpips/loss/lpips.py (LPIPS().eval(), CPU fp32, validation_step order: "
                              "lpips(gt, pred))"},
           "cases": CASES, "terms": [], "lpips": []}
    with torch.no_grad():
        for c in CASES:
            pred, gt = O.pair_inputs(c["n"], c["H"], c["W"], c["seed"])
            terms, val = reference_terms(ns, model, gt, pred)
            t_o = O.layer_terms(sd, gt, pred)
            v_o = O.lpips(sd, gt, pred)
            e_t = ((t_o - terms).abs() / terms.abs().clamp(min=1e-6)).max().item()
            e_v = ((v_o - val).abs() / val.abs()).max().item()
            print(f"{c}: lpips {val.tolist()}  oracle rel err: terms {e_t:.2e}  total {e_v:.2e}")
            assert e_t < 1e-5 and e_v < 1e-5, (e_t, e_v)
            assert 0.05 < val.min() and val.max() < 0.5, val
            out["terms"].append(terms)
            out["lpips"].append(val)
    torch.save(out, os.path.join(GOLD, "lpips.pt"))
    with open(os.path.join(GOLD, "lpips_keys.json"), "w") as f:
        f.write("[\n" + ",\n".join(json.dumps(k) for k in keys) + "\n]\n")
    print(f"wrote {GOLD}/lpips.pt and lpips_keys.json ({len(keys)} keys)")


if __name__ == "__main__":
    main()
