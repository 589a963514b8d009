"""Summarise ncu captures (run here, no GPU needed):
    python tools/ncu_summary.py <name> <rep.ncu-rep> [launch_list.csv]  ->  profiles/ncu_<name>.md (+ ncu_summary.json entry)
"""
import csv, io, json, os, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
        "dram__cycles_active.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "launch__registers_per_thread", "launch__shared_mem_per_block_dynamic", "launch__grid_size", "launch__block_size",
        "sm__inst_executed.avg.per_cycle_elapsed", "smsp__cycles_elapsed.avg.per_second", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "lts__t_bytes.sum", "l1tex__t_bytes_pipe_lsu_mem_global_op_st.sum", "l1tex__t_bytes_pipe_lsu_mem_global_op_ld.sum"]


def raw(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    res = []
    for r in rows[2:]:
        d = {}
        for h, u, v in zip(hdr, units, r):
            if h in KEYS or h in ("Kernel Name",):
                d[h] = (v, u)
        res.append(d)
    return res


def stalls(rep):
    out = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    if len(rows) < 3:
        return {}
    hdr, data = rows[1], rows[2:]
    ci = {h: i for i, h in enumerate(hdr)}
    st = [h for h in hdr if h.startswith("stall_") and "Not Issued" not in h]
    def num(x):
        try:
            return float(x or 0)
        except ValueError:      # a repeated header row (several kernels in one report)
            return 0.0
    agg = {s: sum(num(r[ci[s]]) for r in data if len(r) > ci[s]) for s in st}
    tot = sum(agg.values()) or 1.0
    return {k: round(100 * v / tot, 1) for k, v in sorted(agg.items(), key=lambda x: -x[1]) if v > 0}


def to_bytes(v, u):
    f = float(v.replace(",", ""))
    mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
    return f * mult


def main():
    name, rep = sys.argv[1], sys.argv[2]
    launches = sys.argv[3] if len(sys.argv) > 3 else None
    ks = raw(rep)
    lines = ["# ncu summary: %s" % name, "", "source report: `%s` (ncu --set full --clock-control none --import-source on)" % os.path.basename(rep), ""]
    summ = {}
    for d in ks:
        kn = d.get("Kernel Name", ("?", ""))[0]
        lines.append("## %s" % kn[:120])
        lines.append("")
        lines.append("| metric | value | unit |")
        lines.append("|---|---|---|")
        for k in KEYS:
            if k in d:
                lines.append("| %s | %s | %s |" % (k, d[k][0], d[k][1]))
        rd = to_bytes(*d["dram__bytes_read.sum"]) if "dram__bytes_read.sum" in d else None
        wr = to_bytes(*d["dram__bytes_write.sum"]) if "dram__bytes_write.sum" in d else None
        if rd is not None:
            lines.append("| dram read+write per launch | %.1f | MB |" % ((rd + wr) / 1e6))
            summ = {"dram_bytes_per_launch": rd + wr, "dram_read": rd, "dram_write": wr,
                    "duration_us_under_ncu": float(d["gpu__time_duration.sum"][0].replace(",", "")) * ({"us": 1, "ms": 1e3, "ns": 1e-3}.get(d["gpu__time_duration.sum"][1], 1)),
                    "kernel": kn[:80]}
        lines.append("")
    s = stalls(rep)
    if s:
        lines += ["warp-stall sampling, share of samples by reason (all instructions): `%s`" % json.dumps(s), ""]
    if launches and os.path.exists(launches):
        lines += ["## launch list (`ncu --metrics gpu__time_duration.sum --clock-control none`, cold-cache, serialised)", "",
                  "| kernel | launches | mean us | share of profiled GPU time |", "|---|---|---|---|"]
        agg = {}
        for r in csv.reader(open(launches)):
            if len(r) > 10 and r[-3] == "gpu__time_duration.sum":
                kn = r[4].split("(")[0][:90]
                ns = float(r[-1].replace(",", "")) * ({"ns": 1, "us": 1e3, "usecond": 1e3, "msecond": 1e6, "nsecond": 1}.get(r[-2], 1))
                a = agg.setdefault(kn, [0, 0.0])
                a[0] += 1
                a[1] += ns
        tot = sum(v[1] for v in agg.values()) or 1
        for kn, (c, ns) in sorted(agg.items(), key=lambda x: -x[1][1])[:14]:
            lines.append("| %s | %d | %.2f | %.1f%% |" % (kn, c, ns / c / 1e3, 100 * ns / tot))
        lines.append("")
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    open(os.path.join(ROOT, "profiles", "ncu_%s.md" % name), "w").write("\n".join(lines))
    sj = os.path.join(ROOT, "profiles", "ncu_summary.json")
    allj = json.load(open(sj)) if os.path.exists(sj) else {}
    allj[name.split("_")[-1] if name.split("_")[-1] in ("c2", "c3", "c4", "c5mb") else name] = summ
    json.dump(allj, open(sj, "w"), indent=1)
    print("\n".join(lines[:40]))


if __name__ == "__main__":
    main()
