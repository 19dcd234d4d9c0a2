"""One line per profiled launch from an `ncu --set full` report: time, DRAM bytes, tensor-pipe activity, L2 -> SM traffic,
L2 hit rate, grid, registers, local-memory (spill) instructions, SM clock.

  ncu -i x.ncu-rep --page raw --csv > /tmp/raw.csv
  python tools/ncu_summary.py /tmp/raw.csv [--labels qkv_fwd,out_fwd,...] [--out gemm_ncu_summary.txt]"""
import argparse
import csv

COLS = [("gpu__time_duration.sum", "time"), ("dram__bytes_read.sum", "dramR"), ("dram__bytes_write.sum", "dramW"),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor%active"),
        ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed", "tensor%elapsed"),
        ("l1tex__m_xbar2l1tex_read_bytes.sum.per_second", "L2->SM"), ("lts__t_sector_hit_rate.pct", "L2hit%"),
        ("launch__grid_size", "grid"), ("launch__registers_per_thread", "regs"),
        ("sass__inst_executed_local_loads", "LDL"), ("sass__inst_executed_local_stores", "STL"),
        ("sm__cycles_elapsed.avg.per_second", "SMclk")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--labels", default="")
    ap.add_argument("--out", default=None)
    ap.add_argument("--header", default="")
    a = ap.parse_args()
    rows = list(csv.reader(open(a.csv)))
    hdr, units, body = rows[0], rows[1], rows[2:]
    ix = {h: i for i, h in enumerate(hdr)}
    labels = a.labels.split(",") if a.labels else []
    out = [a.header] if a.header else []
    for n, r in enumerate(body):
        name = r[ix["Kernel Name"]]
        name = name[:name.index("(")] if "(" in name else name
        parts = [f"{(labels[n] if n < len(labels) else ''):14s} {name[:44]:44s}"]
        for col, short in COLS:
            if col in ix:
                v, u = r[ix[col]], units[ix[col]]
                try:
                    v = f"{float(v.replace(',', '')):.4g}"
                except ValueError:
                    pass
                parts.append(f"{short}={v}{u}")
        out.append(" | ".join(parts))
    text = "\n".join(out) + "\n"
    if a.out:
        open(a.out, "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
