"""Summarise an ncu launch list (CSV of `ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum
--csv ...`) into a per-kernel table, and (with --traffic-json) the per-launch DRAM traffic of the GEMM core that
bench.py reports as `roofline.traffic`.

  python tools/summarise_launches.py launches.csv --out launches_summary.txt \
         --traffic-json gemm_dram_traffic.json"""
import argparse
import collections
import csv
import json
import re


def load(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    ids = collections.OrderedDict()
    for x in csv.DictReader(lines):
        k = x["ID"]
        name = re.sub(r"\(.*", "", x["Kernel Name"]).replace("void ", "").replace("mb200::", "")
        d = ids.setdefault(k, {"name": name, "grid": x.get("Grid Size", "")})
        v = float(x["Metric Value"].replace(",", ""))
        unit = x["Metric Unit"]
        m = x["Metric Name"]
        if m == "gpu__time_duration.sum":
            v *= {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}.get(unit, 1e-3)
        elif m.startswith("dram__bytes"):
            v *= {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1.0)
        d[m] = v
    return list(ids.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--out", default=None)
    ap.add_argument("--traffic-json", default=None)
    ap.add_argument("--note", default="")
    a = ap.parse_args()
    L = load(a.csv)
    per = collections.OrderedDict()
    tot = 0.0
    for v in L:
        t = v.get("gpu__time_duration.sum", 0.0)
        p = per.setdefault(v["name"], [0, 0.0, 0.0, 0.0])
        p[0] += 1
        p[1] += t
        p[2] += v.get("dram__bytes_read.sum", 0.0)
        p[3] += v.get("dram__bytes_write.sum", 0.0)
        tot += t
    lines = [f"{len(L)} launches, total kernel time {tot:.1f} us (ncu: serialised, cold cache, PDL overlap not visible)"
             + (f" — {a.note}" if a.note else "")]
    for n, (c, t, r, w) in sorted(per.items(), key=lambda kv: -kv[1][1]):
        lines.append(f"{t:10.1f} us {100 * t / tot:5.1f}%  n={c:4d}  avg={t / c:8.1f}us  dramR={r / 1e6:9.1f}MB dramW={w / 1e6:9.1f}MB  {n[:100]}")
    text = "\n".join(lines) + "\n"
    print(text)
    if a.out:
        open(a.out, "w").write(text)
    if a.traffic_json:
        g = [v for v in L if "gemm" in v["name"] and "wgmma" in v["name"]]
        if g:
            b = sum(v.get("dram__bytes_read.sum", 0.0) + v.get("dram__bytes_write.sum", 0.0) for v in g)
            json.dump({"bytes_per_launch": b / len(g), "gemm_launches": len(g), "total_dram_bytes": b,
                       "source": a.csv, "note": a.note or "dram__bytes_read.sum + dram__bytes_write.sum over every "
                       "gemm_wgmma_kernel launch of one profiled train step / number of those launches"},
                      open(a.traffic_json, "w"), indent=1)


if __name__ == "__main__":
    main()
