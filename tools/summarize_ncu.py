"""Turn ncu outputs into small text/CSV summaries.

  python tools/summarize_ncu.py launches launches.csv launches_summary.csv
  python tools/summarize_ncu.py full prof_conv.ncu-rep ncu_prof_conv.txt [kernel-substring]
"""
import csv, io, re, subprocess, sys
from collections import defaultdict

KEEP = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_tensor.sum", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts_mem_shared.sum", "launch__registers_per_thread",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "launch__shared_mem_per_block_dynamic", "launch__block_size", "launch__grid_size", "launch__cluster_dim_x",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
]


def launches(src, dst):
    rows = []
    with open(src) as f:
        lines = [l for l in f if not l.startswith("==")]
    rd = csv.DictReader(io.StringIO("".join(lines)))
    for r in rd:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        v = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "ns")
        ms = v * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(unit, 1e-6)
        name = re.sub(r"\(.*", "", r["Kernel Name"])
        rows.append((name, ms))
    tot = sum(m for _, m in rows)
    agg = defaultdict(lambda: [0, 0.0])
    for n, m in rows:
        agg[n][0] += 1
        agg[n][1] += m
    with open(dst, "w") as f:
        f.write("# ncu launch list summary: `ncu --metrics gpu__time_duration.sum --clock-control none -c 3500 python bench.py "
                "--steps 1 --warmup 0 --profile-run`\n")
        f.write(f"# first {len(rows)} launches of one clip (setup + the first CFG sampler steps); serialised, cold-cache times: "
                f"compare SHARES. total {tot:.1f} ms\n")
        f.write("kernel,launches,ms,share\n")
        for n, (c, m) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
            f.write(f"{n},{c},{m:.2f},{m / tot:.4f}\n")
    print(open(dst).read())


def full(src, dst, pat=None):
    out = subprocess.run(["ncu", "-i", src, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rd = list(csv.reader(io.StringIO(out)))
    hdr, units = rd[0], rd[1]
    body = rd[2:]
    ki = hdr.index("Kernel Name")
    sel = [r for r in body if pat is None or pat in r[ki]]
    r = sel[-1]
    with open(dst, "w") as f:
        f.write(f"Kernel Name = {r[ki]} \n")
        for k in KEEP:
            if k in hdr:
                i = hdr.index(k)
                f.write(f"{k} = {r[i]} {units[i]}\n")
    print(open(dst).read())


if __name__ == "__main__":
    if sys.argv[1] == "launches":
        launches(sys.argv[2], sys.argv[3])
    else:
        full(sys.argv[2], sys.argv[3], sys.argv[4] if len(sys.argv) > 4 else None)
