"""Per-shape bound model of the tensor-core ops of one CFG forward, against the CUDA-event times of tools/prof_forward.py
(`python tools/roofline_model.py <file>` with the output of tools/prof_forward.py).

For every `tc M.. N.. K..` line: time at the tensor bound (measured burst bf16 peak), at the L2->SM operand-traffic bound (TMA chip
throughput) and at the HBM bound (algorithmic bytes / measured copy peak),
using the tile widths of gcd_tc_run for large problems (BN 256/160/128) and the operand traffic of its tiles (64 rows for ops with a residual or an fp32 output, else 128): every tile reads its own
activation rows and BN x K weight rows from L2."""
import json, os, re, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
# without MEASURED_PEAKS.json: H100 SXM data sheet (dense 16-bit, 700 W card; HBM3), not measured
TENSOR = pk.get("bf16_tflops", 989.0) * 1e12
HBM = pk.get("hbm_gbs", 3350.0) * 1e9
L2SM = 5.5e12          # published L2 read bandwidth of H100 (5.5 - 7 TB/s), not measured here
rx = re.compile(r"\s*([\d.]+) ms\s+x\s*(\d+)\s+(\d+) TF.*tc M(\d+) N(\d+) K(\d+) taps(\d+) g(\d) r(\d)(\d) o(\d)")
rows = []
section = None
SRC = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "profiles", "r2_prof_forward_final.txt")
for line in open(SRC):
    if line.startswith("=="):
        section = line.split(":")[0].strip("= ")
    m = rx.match(line)
    if not m:
        continue
    ms, cnt, tf, M, N, K, taps, g, r1, r2, o = m.groups()
    ms, cnt, M, N, K, taps = float(ms), int(cnt), int(M), int(N), int(K), int(taps)
    g, r1, r2, o = int(g), int(r1), int(r2), int(o)
    BN = 256 if (N % 256 == 0 or N >= 384) else (160 if N % 160 == 0 else 128)
    ntile = -(-N // BN)
    a_bytes = M * K * 2 * ntile                                  # every N-tile pass re-reads its A tiles from L2
    tile_m = 64 if (r1 or r2 or o) and not g else 128            # gcd_tc_run: ping-pong schedule for these epilogues
    b_bytes = M / tile_m * ntile * BN * K * 2                    # every tile reads the BN weight rows of its N-tile
    t_l2 = (a_bytes + b_bytes) / L2SM
    t_tc = 2.0 * M * N * K / TENSOR
    nout = N // 2 if g else N
    hbm = M * (K // taps) * 2 + M * nout * (4 if o else 2) + (r1 + r2) * M * N * 4     # fp32 residuals on the path
    t_hbm = hbm / HBM
    t = ms / cnt * 1e-3
    bound = max((t_tc, "tensor"), (t_l2, "L2->SM"), (t_hbm, "HBM"))
    rows.append((section, ms, cnt, M, N, K, taps, BN, t * 1e6, t_tc * 1e6, t_l2 * 1e6, t_hbm * 1e6, bound[1], bound[0] / t))
print(f"{'section':12s} {'ms':>7s} {'x':>4s} {'M':>8s} {'N':>6s} {'K':>6s} BN  {'us/launch':>9s} {'tensor':>8s} {'L2->SM':>8s} {'HBM':>8s}  binding  frac-of-bound")
for r in sorted(rows, key=lambda r: -r[1]):
    print(f"{r[0]:12s} {r[1]:7.2f} {r[2]:4d} {r[3]:8d} {r[4]:6d} {r[5]:6d} {r[7]:3d}  {r[8]:9.1f} {r[9]:8.1f} {r[10]:8.1f} {r[11]:8.1f}  {r[12]:7s}  {r[13]:.2f}")
tot = sum(r[1] for r in rows)
low = sum(r[1] * (1 - min(1.0, r[13])) for r in rows)
print(f"\nlisted tensor-core time {tot:.1f} ms; time above the binding bound {low:.1f} ms ({100 * low / tot:.0f} %)")
