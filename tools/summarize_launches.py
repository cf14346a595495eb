"""ncu --csv launch list (gpu__time_duration.sum [+ dram__bytes_read.sum, dram__bytes_write.sum]) of ONE train step ->
markdown table per kernel (launches, total us, share, DRAM GB, GB/s) + optional traffic json.

    python tools/summarize_launches.py step_launches.csv launches.md [traffic.json]
"""
import collections
import csv
import json
import re
import sys

src, dst = sys.argv[1], sys.argv[2]
lines = [ln for ln in open(src) if not ln.startswith("==")]
rows = list(csv.reader(lines))
hdr = rows[0]
ki, mi, ui, vi, ii = (hdr.index(k) for k in ("Kernel Name", "Metric Name", "Metric Unit", "Metric Value", "ID"))
scale = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1, "ms": 1e3, "usecond": 1, "nsecond": 1e-3, "msecond": 1e3}
agg = collections.defaultdict(lambda: {"ids": set(), "rd": 0.0, "wr": 0.0, "us": 0.0})
for r in rows[1:]:
    if len(r) <= vi:
        continue
    name = re.sub(r"\(.*", "", r[ki]).replace("<unnamed>::", "").replace("void ", "").strip()
    name = re.sub(r"^at::native::", "at::", name)[:90]
    v = float(r[vi].replace(",", "")) * scale.get(r[ui], 1)
    a = agg[name]
    a["ids"].add(r[ii])
    if r[mi] == "dram__bytes_read.sum":
        a["rd"] += v
    elif r[mi] == "dram__bytes_write.sum":
        a["wr"] += v
    elif r[mi] == "gpu__time_duration.sum":
        a["us"] += v
tot = sum(a["us"] for a in agg.values())
out = [f"| kernel | launches | total µs | share | DRAM GB (r+w) | GB/s |", "|---|---:|---:|---:|---:|---:|"]
for name, a in sorted(agg.items(), key=lambda kv: -kv[1]["us"]):
    gb = (a["rd"] + a["wr"]) / 1e9
    out.append(f"| `{name}` | {len(a['ids'])} | {a['us']:.0f} | {100 * a['us'] / tot:.1f}% | {gb:.3f} | {gb / max(a['us'], 1e-9) * 1e6:.0f} |")
head = sys.argv[4] if len(sys.argv) > 4 else ""
open(dst, "w").write(f"{head}\n\nTotal {tot / 1e3:.2f} ms over {sum(len(a['ids']) for a in agg.values())} launches (per-launch times are "
                     f"serialised / cold-cache under ncu: SHARES are meaningful, not the absolute sum).\n\n" + "\n".join(out) + "\n")
print("\n".join(out[:24]))
if len(sys.argv) > 3 and sys.argv[3] != "-":
    json.dump({"source": "ncu dram__bytes_read.sum + dram__bytes_write.sum + gpu__time_duration.sum, one eager train step",
               "kernels": {k: {"launches": len(v["ids"]), "dram_read_bytes": v["rd"], "dram_write_bytes": v["wr"],
                               "time_us_under_ncu": v["us"]} for k, v in agg.items()}}, open(sys.argv[3], "w"), indent=1)
