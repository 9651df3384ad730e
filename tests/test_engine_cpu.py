"""CPU tests of the plumbing the execution engines share (gcd_b200/engine.py): the packed-engine cache key and the GroupNorm
statistics arena."""
import gzip
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, "tests", "golden")

from gcd_b200 import spec, synthetic  # noqa: E402


# ------------------------------------------------------------------------------------------- weight (re)load / EMA swap
def test_engine_key_sees_data_copy_and_litema_shadows_every_parameter():
    """ADVICE r1: `param.data.copy_` (what the reference's LitEma.copy_to / restore do, modules/ema.py) does not bump
    `_version`; the engine cache key must still change, and LitEma must find parameters to shadow (requires_grad)."""
    from gcd_b200.engine import weights_key
    from gcd_b200.unet import VideoUNet
    net = VideoUNet(**spec.unet_ctor_kwargs(spec.UNET_TINY))
    net.load_state_dict(synthetic.seeded_state(spec.unet_param_shapes(spec.UNET_TINY), seed=0))
    k0 = weights_key(net, "cpu")
    assert weights_key(net, "cpu") == k0
    other = synthetic.seeded_state(spec.unet_param_shapes(spec.UNET_TINY), seed=5)
    with torch.no_grad():
        for name, p in net.named_parameters():
            v = p._version
            p.data.copy_(other[name])
            assert p._version == v                      # the blind spot the content probe covers
    assert weights_key(net, "cpu") != k0
    n_params = sum(1 for _ in net.parameters())
    assert all(p.requires_grad for p in net.parameters())
    # the reference's LitEma shadows every parameter that requires grad, under its own buffer naming (golden: its
    # m_name2s_name for this network, oracle/pin_against_reference.py) => `model_ema.*` checkpoint keys load
    gold = json.load(gzip.open(os.path.join(GOLD, "ref_ema_conditioner.json.gz"), "rt"))["litema_unet_tiny"]
    from gcd_b200 import checkpoint
    assert len(gold) == n_params
    assert {n: checkpoint.ema_key(n) for n, p in net.named_parameters() if p.requires_grad} == gold
    # LitEma.copy_to / restore write the shadows with `param.data.copy_` (ema_scope entry / exit, models/diffusion.py)
    k1 = weights_key(net, "cpu")
    stored = [p.detach().clone() for p in net.parameters()]
    with torch.no_grad():
        for p in net.parameters():
            p.data.copy_(p.data * 0.5)
    assert weights_key(net, "cpu") != k1
    with torch.no_grad():
        for p, v in zip(net.parameters(), stored):
            p.data.copy_(v)
    assert weights_key(net, "cpu") == k1


def test_stats_arena_slots_and_growth():
    """GroupNorm statistics arena (engine.StatsArena): one memset per forward, one slot per producer, slot size follows the batch."""
    from gcd_b200 import engine as U

    class Pool:
        def __init__(self):
            self.bufs = {}

        def get(self, name, shape, dtype):
            return self.bufs.setdefault((name, tuple(shape), dtype), torch.zeros(shape, dtype=dtype))

    zeroed = []
    orig = U.ops.zero_tensor
    U.ops.zero_tensor = lambda t: (zeroed.append(t.numel()), t.zero_())
    try:
        a = U.StatsArena(Pool())
        a.reset(28)
        s0, s1 = a.take(28), a.take(2)
        assert s0.numel() == s1.numel() == 64 * 64 and s0.data_ptr() != s1.data_ptr() and zeroed == [U.StatsArena.SLOTS * 4096]
        s0[:10] = 1.0
        a.reset(28)                                            # next forward: same storage, zeroed again by ONE memset
        assert a.take(28).data_ptr() == s0.data_ptr() and float(s0.sum()) == 0.0 and len(zeroed) == 2
        a.reset(200)                                           # bigger batch -> bigger slots
        assert a.take(200).numel() == 200 * 64
        with pytest.raises(AssertionError):
            a.take(500)
    finally:
        U.ops.zero_tensor = orig
