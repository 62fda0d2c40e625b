"""Summarise `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --csv` launch lists of one eager
train step per model (tests/probes/ncu_step.py) into per-kernel-class DRAM traffic / time tables.

    python tests/probes/summarize_traffic.py gpurun_out/r2a profiles/r2_traffic   # writes *_summary.json + *.md
"""
import csv, gzip, io, json, os, re, sys
from collections import defaultdict

src, dst = sys.argv[1], sys.argv[2]
UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3,
        "nsecond": 1e-3, "second": 1e6}
LEG = {"slowfast": "slowfast", "mvit": "mvitv2_s", "x3d": "x3d_m"}
summary, md = {}, []
for which in ("slowfast", "mvit", "x3d"):
    path = os.path.join(src, f"traffic_{which}.csv")
    if not os.path.exists(path):
        continue
    lines = [l for l in open(path) if not l.startswith("==")]
    rows = list(csv.DictReader(io.StringIO("".join(lines))))
    per = defaultdict(lambda: defaultdict(float))
    ids = defaultdict(set)
    for r in rows:
        name = re.sub(r"\(.*$", "", r["Kernel Name"]).strip()
        name = re.sub(r"^void ", "", name)
        val = float(r["Metric Value"].replace(",", "")) * UNIT.get(r["Metric Unit"], 1.0)
        per[name][r["Metric Name"]] += val
        ids[name].add(r["ID"])
    total_us = sum(v["gpu__time_duration.sum"] for v in per.values())
    table = []
    for name, v in sorted(per.items(), key=lambda kv: -kv[1]["gpu__time_duration.sum"]):
        n = len(ids[name])
        rd, wr, us = v["dram__bytes_read.sum"], v["dram__bytes_write.sum"], v["gpu__time_duration.sum"]
        table.append(dict(kernel=name, launches=n, total_us=round(us, 1), share=round(us / total_us, 4),
                          dram_read_mb=round(rd / 1e6, 1), dram_write_mb=round(wr / 1e6, 1),
                          dram_bytes_per_launch=(rd + wr) / n, dram_gbs=round((rd + wr) / us / 1e3, 1)))
    leg = {}
    for t in table:
        short = t["kernel"].split("<")[0].replace("sfb::", "").replace("_kernel", "")
        if short not in leg:
            leg[short] = dict(dram_bytes_per_launch=t["dram_bytes_per_launch"], launches=t["launches"],
                              dram_gbs_under_ncu=t["dram_gbs"],
                              source=f"profiles/{os.path.basename(dst)}_{which}.csv.gz (ncu dram__bytes_read.sum + "
                                     f"dram__bytes_write.sum, one eager step, all launches of the class)")
    summary[LEG[which]] = leg
    md.append(f"## {which}: one eager train step under ncu ({len(rows) // 3} launches, {total_us / 1e3:.1f} ms serialised)\n")
    md.append("| kernel | launches | total us | share | DRAM read MB | DRAM write MB | DRAM GB/s (under ncu) |")
    md.append("|---|---:|---:|---:|---:|---:|---:|")
    for t in table[:28]:
        md.append(f"| `{t['kernel'][:70]}` | {t['launches']} | {t['total_us']:.0f} | {100 * t['share']:.1f}% | "
                  f"{t['dram_read_mb']:.0f} | {t['dram_write_mb']:.0f} | {t['dram_gbs']:.0f} |")
    md.append("")
    with gzip.open(f"{dst}_{which}.csv.gz", "wt") as f:
        f.write("".join(lines))
json.dump(summary, open(f"{dst}_summary.json", "w"), indent=1)
open(f"{dst}.md", "w").write(
    "# Round 2 - DRAM traffic per kernel class (ncu `dram__bytes_read.sum`, `dram__bytes_write.sum`, `gpu__time_duration.sum`)\n\n"
    "Command (per model): `ncu --profile-from-start off --metrics gpu__time_duration.sum,dram__bytes_read.sum,"
    "dram__bytes_write.sum --clock-control none --csv --log-file ... python tests/probes/ncu_step.py <model>` - one eager train step "
    "(fwd + CE + bwd) after two warm-up steps, parity mode, recipe batch.  Times under ncu are serialised and cold-cache: compare "
    "shares; the DRAM byte counts are what `bench.py`'s `roofline.traffic` reports (bytes per launch of the dominant class).\n\n"
    + "\n".join(md))
print(json.dumps({k: {kk: round(vv["dram_bytes_per_launch"] / 1e6, 2) for kk, vv in list(v.items())[:6]} for k, v in summary.items()}))
