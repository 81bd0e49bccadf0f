"""Summarise an ncu launch list (csv from `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum
--clock-control none --csv ...`) of `bench.py --steps 1 --warmup 1`: one optimizer step = the launches between the last two
adamw_kernel launches.  Writes the per-kernel table and the GEMM DRAM traffic json used by bench.py's roofline.traffic.

    python tools/summarize_launches.py $MIDI_TOOLS_OUT/launches.csv $MIDI_TOOLS_OUT/run
"""
import csv
import json
import re
import sys
from collections import defaultdict


def main():
    src, prefix = sys.argv[1], sys.argv[2]
    rows = []
    with open(src, newline="") as f:
        lines = [l for l in f if l.startswith('"')]
    rd = csv.DictReader(lines)
    per = {}
    for r in rd:
        key = r["ID"]
        ent = per.setdefault(key, {"name": r["Kernel Name"], "t": 0.0, "rd": 0.0, "wr": 0.0})
        val = float(r["Metric Value"].replace(",", "")) if r["Metric Value"] not in ("", "n/a") else 0.0
        unit = r["Metric Unit"]
        m = r["Metric Name"]
        scale = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6, "byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1.0)
        if m.startswith("gpu__time_duration"):
            ent["t"] = val * scale
        elif m.startswith("dram__bytes_read"):
            ent["rd"] = val * scale
        elif m.startswith("dram__bytes_write"):
            ent["wr"] = val * scale
    launches = [per[k] for k in sorted(per, key=lambda x: int(x))]
    idx = [i for i, l in enumerate(launches) if "adamw_kernel" in l["name"]]
    if len(idx) >= 2:
        launches = launches[idx[-2] + 1: idx[-1] + 1]
    agg = defaultdict(lambda: [0, 0.0, 0.0])
    for l in launches:
        n = re.sub(r"\(.*", "", l["name"]).replace("void ", "").replace("<unnamed>::", "")
        a = agg[n]
        a[0] += 1
        a[1] += l["t"]
        a[2] += l["rd"] + l["wr"]
    tot = sum(a[1] for a in agg.values())
    out = [f"one optimizer step: {len(launches)} launches, sum of kernel times {tot / 1e3:.2f} ms (cold-cache, serialised under ncu)",
           f"{'kernel':60s} {'launches':>8s} {'time(us)':>10s} {'share':>7s} {'dram GB':>9s}"]
    for n, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        if a[1] / tot < 0.001:
            continue
        out.append(f"{n[:60]:60s} {a[0]:8d} {a[1]:10.1f} {a[1] / tot:7.1%} {a[2] / 1e9:9.2f}")
    gemm = [a for n, a in agg.items() if "gemm_wgmma_kernel" in n]
    g_l, g_t, g_b = sum(a[0] for a in gemm), sum(a[1] for a in gemm), sum(a[2] for a in gemm)
    out.append(f"GEMM share of the step: {g_t / 1e3:.2f} ms of {tot / 1e3:.2f} ms = {g_t / tot:.1%}; {g_l} launches, {g_b / 1e9:.1f} GB DRAM")
    open(prefix + "_launches_step_summary.txt", "w").write("\n".join(out) + "\n")
    json.dump({"kernel": "gemm_wgmma_kernel", "launches_per_step": g_l, "dram_bytes_per_step": g_b,
               "dram_bytes_per_launch": g_b / max(g_l, 1),
               "source": f"{src} (ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none "
                         "python bench.py --steps 1 --warmup 1 --no-cpu-baseline --no-generate --no-hbm-kernels; one optimizer step)"},
              open(prefix + "_gemm_traffic.json", "w"), indent=1)
    print("\n".join(out))


if __name__ == "__main__":
    main()
