"""Pivot an ncu launch list (`ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none --csv
--log-file raw.csv <command>`) into one row per launch, keep the LAST decode step (from the last embedding gather to the end), and print a
per-kernel table.  With --traffic the DRAM bytes per mat-vec launch are written as json (bench.py reads it for roofline.traffic).
usage: python tools/launch_list.py raw.csv out.csv [--traffic traffic.json] [--all]"""
import csv, sys, json, collections, re

def main():
    raw, out = sys.argv[1], sys.argv[2]
    traffic = sys.argv[sys.argv.index("--traffic") + 1] if "--traffic" in sys.argv else None
    rows = [r for r in csv.reader(open(raw, errors="replace")) if len(r) > 10]
    hdr = next(r for r in rows if r[0] == "ID")
    ix = {h: i for i, h in enumerate(hdr)}
    launches = collections.OrderedDict()
    for r in rows:
        if r[0] == "ID" or not r[0].isdigit():
            continue
        L = launches.setdefault(int(r[0]), dict(id=int(r[0]), stream=r[ix["Stream"]], kernel=r[ix["Kernel Name"]], grid=r[ix["Grid Size"]], block=r[ix["Block Size"]]))
        v = float(r[ix["Metric Value"]].replace(",", ""))
        unit = r[ix["Metric Unit"]]
        name = r[ix["Metric Name"]]
        if name == "gpu__time_duration.sum":
            v *= {"ns": 1, "us": 1e3, "ms": 1e6, "s": 1e9}.get(unit, 1)
        else:
            v *= {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
        L[name] = v
    ls = list(launches.values())
    if "--all" not in sys.argv:
        starts = [i for i, L in enumerate(ls) if "dequant_rows_kernel" in L["kernel"]]
        if len(starts) >= 2:
            ls = ls[starts[-2]:starts[-1]]          # the last COMPLETE step (the capture limit may cut the final one short)
        elif starts:
            ls = ls[starts[-1]:]
    with open(out, "w") as f:
        f.write('"# %s ; launches %d..%d ; cold-cache, serialised (ncu)"\n' % (" ".join(sys.argv), ls[0]["id"], ls[-1]["id"]))
        w = csv.writer(f)
        w.writerow(["ncu_id", "stream", "kernel", "grid", "block", "gpu__time_duration.sum [ns]", "dram__bytes_read.sum [B]", "dram__bytes_write.sum [B]"])
        for L in ls:
            w.writerow([L["id"], L["stream"], L["kernel"][:90], L["grid"], L["block"], int(L.get("gpu__time_duration.sum", 0)),
                        int(L.get("dram__bytes_read.sum", 0)), int(L.get("dram__bytes_write.sum", 0))])
    agg = collections.OrderedDict()
    for L in ls:
        key = re.sub(r"\(.*", "", L["kernel"]) + " " + L["grid"] + "x" + L["block"]
        a = agg.setdefault(key, [0, 0.0, 0.0])
        a[0] += 1; a[1] += L.get("gpu__time_duration.sum", 0); a[2] += L.get("dram__bytes_read.sum", 0) + L.get("dram__bytes_write.sum", 0)
    tot = sum(a[1] for a in agg.values())
    print("| kernel grid x block | launches | total us | share | avg us | DRAM MB / launch |\n|---|---|---|---|---|---|")
    for k, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("| `%s` | %d | %.1f | %.1f %% | %.2f | %.2f |" % (k, a[0], a[1] / 1e3, 100 * a[1] / tot, a[1] / a[0] / 1e3, a[2] / a[0] / 1e6))
    print("total %.1f us over %d launches" % (tot / 1e3, len(ls)))
    if traffic:
        mv = [L for L in ls if "mmv_fast_kernel" in L["kernel"] or "mmv_kernel" in L["kernel"]]
        b = sum(L.get("dram__bytes_read.sum", 0) + L.get("dram__bytes_write.sum", 0) for L in mv)
        json.dump({"source": "%s (ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum, one decode step of bench.py)" % out,
                   "matvec_launches_per_step": len(mv), "dram_bytes_per_matvec_launch": b / max(1, len(mv)), "dram_bytes_matvecs_per_step": b},
                  open(traffic, "w"), indent=1)

if __name__ == "__main__":
    main()
