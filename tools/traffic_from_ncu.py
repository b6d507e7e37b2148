"""Per-kernel and per-stage DRAM traffic of ONE pipeline step (tools/step_once.py), from the CSV of
`ncu -i X.ncu-rep --page raw --csv`:

    python tools/traffic_from_ncu.py <ncu.csv> <out.json> <V> <T>

per kernel DRAM bytes + cold duration, per stage the sums next to the algorithmic bytes."""
import csv, json, sys
src, out, V, T = sys.argv[1], sys.argv[2], int(sys.argv[3]), int(sys.argv[4])
N = 512 ** 3
rows = list(csv.reader(open(src)))
hdr = rows[0]
ix = {k: hdr.index(k) for k in ("Kernel Name", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum")}
units = rows[1]
def to_bytes(v, u):
    return float(v) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[u]
def to_us(v, u):
    return float(v) * {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}[u]
kern = {}
for r in rows[2:]:
    name = r[ix["Kernel Name"]].split("(")[0].replace("void ", "").replace("<unnamed>::", "")
    k = kern.setdefault(name, {"launches": 0, "dram_read": 0.0, "dram_write": 0.0, "duration_us_cold": 0.0})
    k["launches"] += 1
    k["dram_read"] += to_bytes(r[ix["dram__bytes_read.sum"]], units[ix["dram__bytes_read.sum"]])
    k["dram_write"] += to_bytes(r[ix["dram__bytes_write.sum"]], units[ix["dram__bytes_write.sum"]])
    k["duration_us_cold"] += to_us(r[ix["gpu__time_duration.sum"]], units[ix["gpu__time_duration.sum"]])
stage_of = lambda n: "threshold" if "threshold" in n else ("floodfill" if "k_ff" in n else ("marching_cubes" if "k_mc" in n else None))
alg = {"threshold": 3.0 * N, "floodfill": 4.0 * N, "marching_cubes": 1.0 * N + 12.0 * V + 12.0 * T}
stages = {s: {"traffic": 0.0, "algorithmic": a, "duration_us_cold": 0.0} for s, a in alg.items()}
for n, k in kern.items():
    s = stage_of(n)
    if s:
        stages[s]["traffic"] += k["dram_read"] + k["dram_write"]
        stages[s]["duration_us_cold"] += k["duration_us_cold"]
    for f in ("dram_read", "dram_write", "duration_us_cold"):
        k[f] = round(k[f], 1)
for s in stages.values():
    s["traffic"] = round(s["traffic"], 1); s["duration_us_cold"] = round(s["duration_us_cold"], 1)
    s["traffic_over_algorithmic"] = round(s["traffic"] / s["algorithmic"], 3)
json.dump({"source": f"ncu --set full --clock-control none, one step of tools/step_once.py (512^3 phantom), {src}; cold-cache, "
                     "serialised replays: compare shares, not absolutes",
           "unit": "bytes (dram__bytes_read.sum + dram__bytes_write.sum), microseconds", "V": V, "T": T, "kernels": kern,
           "stages": stages}, open(out, "w"), indent=1)
print(json.dumps(stages, indent=1))
