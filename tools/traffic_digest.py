"""ncu launch-list CSV (tools/frame_once.py under ncu) -> profiles/r2_launches.md + profiles/r2_traffic.json.
Takes the last frame of the list (from its pool_interval_cells_kernel launch to the end)."""
import csv, json, subprocess, sys
from collections import OrderedDict

src, frames = sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 3
rows = [r for r in csv.reader(open(src)) if r and not r[0].startswith("==")]
hdr = rows[0]
ix = {h: i for i, h in enumerate(hdr)}
recs = OrderedDict()
for r in rows[1:]:
    if len(r) < len(hdr):
        continue
    key = r[ix["ID"]]
    d = recs.setdefault(key, {"name": r[ix["Kernel Name"]]})
    val = float(r[ix["Metric Value"]].replace(",", ""))
    unit = r[ix["Metric Unit"]]
    name = r[ix["Metric Name"]]
    if name.startswith("gpu__time_duration"):
        d["us"] = val / 1e3 if unit in ("ns", "nsecond") else (val * 1e3 if unit in ("ms", "msecond") else val)
    else:
        mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
        d[name] = val * mult
launches = list(recs.values())
# one frame = from its first launch (the pooling plan's interval-cell kernel) to the end of the list
starts = [i for i, d in enumerate(launches) if "pool_interval_cells_kernel" in d["name"]]
last = launches[starts[-1]:]
per = len(last)
groups = OrderedDict()
for d in last:
    n = d["name"].split("(")[0].replace("void ", "").replace("bevb200::", "")
    g = groups.setdefault(n, {"launches": 0, "us": 0.0, "bytes": 0.0})
    g["launches"] += 1
    g["us"] += d.get("us", 0.0)
    g["bytes"] += d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)
total_us = sum(g["us"] for g in groups.values())
commit = subprocess.run(["git", "rev-parse", "--short", "HEAD"], capture_output=True, text=True).stdout.strip()
lines = ["# Round 2: one hot-path frame, every launch (ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum",
         "# --clock-control none; cold caches, serialised: compare SHARES, not absolutes).  %d launches, %.1f us, commit %s" % (per, total_us, commit),
         "", "| kernel | launches | us | share | DRAM MB (read + write) |", "|---|---|---|---|---|"]
for n, g in sorted(groups.items(), key=lambda kv: -kv[1]["us"]):
    lines.append("| %s | %d | %.1f | %.1f %% | %.1f |" % (n, g["launches"], g["us"], 100 * g["us"] / total_us, g["bytes"] / 1e6))
open("profiles/r2_launches.md", "w").write("\n".join(lines) + "\n")
def total(pred):
    return sum(g["bytes"] for n, g in groups.items() if pred(n))
out = {"source": "profiles/r2_launches.md (ncu launch list of tools/frame_once.py, commit %s)" % commit,
       "spconv_bytes": total(lambda n: n.startswith("spconv_v6_kernel")),
       "encoder_bytes": total(lambda n: n.startswith(("spconv_v6", "enc_", "rb_", "sparse_to_dense"))),
       "bev_pool_plan_bytes": total(lambda n: n.startswith(("bevpool_fwd_tma", "pool_interval_cells"))),
       "spconv_share_of_frame": round(sum(g["us"] for n, g in groups.items() if n.startswith("spconv_v6_kernel")) / total_us, 4)}
json.dump(out, open("profiles/r2_traffic.json", "w"), indent=1)
print("\n".join(lines[:14]))
print(out)
