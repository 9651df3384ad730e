"""Autotune study of `tc_gemm_kernel`'s tile width / cluster mode per op of the hot path (experiments, on an H100; the cluster-mode argument is ignored by the Hopper kernel).

Records every `gcd_tc_run` descriptor of one full-size CFG forward + one VAE decode, then re-issues each DISTINCT op (same buffers,
same fused epilogue) under every (BN, mode) the kernel supports — `gcd_tc_override` — and times it with CUDA events (median of 7,
back to back; the level-1 operands exceed the L2). Prints, per op, the automatic choice's time, the best configuration and the gain,
and the total over the forward weighted by how often the op occurs. Output: gpurun_out/autotune_tc.json.
"""
import ctypes
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from gcd_b200 import _lib, ops, spec, synthetic  # noqa: E402
from gcd_b200.pipeline import GCDHotPath  # noqa: E402

T, H, W = 14, 72, 128
os.environ["GCD_NO_GRAPH"] = "1"   # eager launches so that gcd_tc_run can be recorded
pipe = GCDHotPath(spec.UNET_KUBRIC, spec.VAE_DECODER, num_steps=1, device="cuda")
pipe.load_state(synthetic.seeded_state(spec.unet_param_shapes(spec.UNET_KUBRIC)), synthetic.seeded_state(spec.decoder_param_shapes(spec.VAE_DECODER)))
x, c, uc, _ = synthetic.seeded_inputs(spec.UNET_KUBRIC, 1, T, H, W)
x, c, uc = x.cuda(), {k: v.cuda() for k, v in c.items()}, {k: v.cuda() for k, v in uc.items()}
z = pipe.sample_latents(x.clone(), c, uc)
pipe.decode_first_stage(z)
torch.cuda.synchronize()

L = ops.lib()
recorded = []
real = L.gcd_tc_run


class _Rec:
    def __call__(self, op_ref, stream):
        op = op_ref._obj
        cp = _lib.TcOp()
        ctypes.memmove(ctypes.byref(cp), ctypes.byref(op), ctypes.sizeof(_lib.TcOp))
        recorded.append(cp)
        return real(op_ref, stream)


L.__dict__["gcd_tc_run"] = _Rec()                  # instance attribute shadows the CDLL function for the recording pass
try:
    z = pipe.sample_latents(x.clone(), c, uc)
    n_unet = len(recorded)
    pipe.decode_first_stage(z)
finally:
    L.__dict__["gcd_tc_run"] = real
torch.cuda.synchronize()


def sig(o):
    e = o.ep
    return (o.Xo * o.Yo * o.Zo, o.N, o.ntaps * o.C, o.ntaps, o.in_mul, int(e.geglu), int(bool(e.res1)), int(bool(e.res2)), int(e.out_f32),
            int(bool(e.rowvec)), int(bool(e.gn_stats)), int(o.w_batch_stride != 0))


groups = {}
for i, o in enumerate(recorded):
    g = groups.setdefault((("unet" if i < n_unet else "vae"),) + sig(o), [o, 0])
    g[1] += 1
st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


SUSTAIN = float(os.environ.get("AUTOTUNE_SECONDS", "0"))     # > 0: time each configuration back to back for this long (power-capped)
TOP = int(os.environ.get("AUTOTUNE_TOP", "0"))               # > 0: only the TOP ops by (burst time x count) of the UNet


def timeit_sustained(o, seconds):
    import time
    for _ in range(20):
        real(ctypes.byref(o), st)
    torch.cuda.synchronize()
    t0 = time.time()
    n = 0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    started = False
    while True:
        el = time.time() - t0
        if not started and el > seconds * 0.4:       # first 40 %: let the clocks settle under the power cap
            a.record(); started = True; n = 0
        if el > seconds:
            break
        for _ in range(20):
            real(ctypes.byref(o), st)
        n += 20
        torch.cuda.synchronize()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / max(n, 1)


def timeit(o, reps=7):
    if SUSTAIN > 0:
        return timeit_sustained(o, SUSTAIN)
    for _ in range(2):
        real(ctypes.byref(o), st)
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); real(ctypes.byref(o), st); real(ctypes.byref(o), st); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / 2)
    ts.sort()
    return ts[len(ts) // 2]


rows, tot_auto, tot_best = [], {"unet": 0.0, "vae": 0.0}, {"unet": 0.0, "vae": 0.0}
order = sorted(groups.items(), key=lambda kv: -kv[1][1])
if TOP > 0:                           # rank the UNet ops by a quick burst timing x count
    sus, SUSTAIN = SUSTAIN, 0.0
    L.gcd_tc_override(0, 0)
    ranked = sorted(((timeit(o, 3) * cnt, key) for key, (o, cnt) in groups.items() if key[0] == "unet" and not key[-1]), reverse=True)
    keep = {k for _, k in ranked[:TOP]}
    order = [(k, v) for k, v in order if k in keep]
    SUSTAIN = sus
for key, (o, cnt) in order:
    if key[-1]:                       # batched weights: single-CTA mode only
        continue
    L.gcd_tc_override(0, 0)
    t_auto = timeit(o)
    best = (t_auto, "auto")
    res = {}
    for bn in ((256,) if key[6] else (128, 160, 256)):
        for mode in (2, 3):
            L.gcd_tc_override(bn, mode)
            rc = real(ctypes.byref(o), st)
            if rc < 0:
                continue
            t = timeit(o)
            res[f"bn{bn}m{mode}"] = round(t, 4)
            if t < best[0]:
                best = (t, f"bn{bn}m{mode}")
    L.gcd_tc_override(0, 0)
    part = key[0]
    tot_auto[part] += t_auto * cnt
    tot_best[part] += best[0] * cnt
    rows.append({"part": part, "M": key[1], "N": key[2], "K": key[3], "taps": key[4], "geglu": key[6], "res": key[7] + key[8], "of32": key[9],
                 "rowvec": key[10], "stats": key[11], "count": cnt, "auto_ms": round(t_auto, 4), "best": best[1], "best_ms": round(best[0], 4),
                 "all": res})
    r = rows[-1]
    print(f"{part} M{r['M']} N{r['N']} K{r['K']} t{r['taps']} g{r['geglu']} r{r['res']} o{r['of32']} rv{r['rowvec']} st{r['stats']} x{cnt}: auto {t_auto:.4f} "
          f"best {best[1]} {best[0]:.4f} ({(1 - best[0] / t_auto) * 100:.1f} %)  {res}", flush=True)
print("totals per pass (ms): auto", tot_auto, "best", tot_best)
os.makedirs("gpurun_out", exist_ok=True)
json.dump({"rows": rows, "total_auto_ms": tot_auto, "total_best_ms": tot_best}, open("gpurun_out/autotune_tc.json", "w"), indent=1)
