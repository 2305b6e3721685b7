"""Turns gpurun_out/*.ncu-rep + the launch-list csv into the tracked summaries under profiles/."""
import collections, csv, io, os, re, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "lts__t_bytes.sum", "l1tex__m_xbar2l1tex_read_bytes.sum",
    "l1tex__m_xbar2l1tex_read_bytes.sum.per_second", "l1tex__data_pipe_tc_wavefronts_mem_shared.sum",
    "TPC.TriageCompute.sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
    "sm__pipe_tensor_cycles_active_realtime.avg.pct_of_peak_sustained_elapsed",
    "sm__mem_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__inst_executed.sum", "sm__cycles_elapsed.avg", "sm__cycles_elapsed.avg.per_second",
]


def raw(rep):
    if rep.endswith(".csv"):  # raw page exported on the GPU box (tools/ncu_capture.sh)
        out = open(rep).read()
    else:
        out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(out)))
    hdr, units = rows[0], rows[1]
    res = []
    for vals in rows[2:]:
        d = {}
        for h, u, v in zip(hdr, units, vals):
            d[h.split(".TriageCompute.")[-1] if ".TriageCompute." in h else h] = (v, u)
        res.append(d)
    return res


def _open(path):
    import gzip
    return gzip.open(path, "rt") if path.endswith(".gz") else open(path)


def launches(path):
    lines = [l for l in _open(path) if not l.startswith("==")]
    tot, cnt = collections.defaultdict(float), collections.Counter()
    for row in csv.DictReader(lines):
        v = float(row["Metric Value"].replace(",", ""))
        v *= {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(row["Metric Unit"], 1e-6)
        name = re.sub(r"\(.*", "", row["Kernel Name"]).replace("void ", "").replace("hvn::", "")
        tot[name] += v
        cnt[name] += 1
    return tot, cnt


def traffic(path):
    """per kernel: launches, summed dram bytes and time of the SECOND (profiled) pass of tools/ncu_target.py"""
    lines = [l for l in open(path) if not l.startswith("==")]
    per = collections.OrderedDict()
    rows = list(csv.DictReader(lines))
    ids = sorted({int(r["ID"]) for r in rows})
    half = ids[len(ids) // 2]  # launches of the warm-up pass come first
    for r in rows:
        if int(r["ID"]) < half:
            continue
        name = re.sub(r"\(.*", "", r["Kernel Name"]).replace("void ", "").replace("hvn::", "")
        name = re.sub(r"<.*", "", name)
        v = float(r["Metric Value"].replace(",", ""))
        u = r["Metric Unit"]
        d = per.setdefault(name, {"ids": set(), "bytes": 0.0, "ms": 0.0})
        d["ids"].add(r["ID"])
        if r["Metric Name"].startswith("dram__bytes"):
            d["bytes"] += v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
        else:
            d["ms"] += v * {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3}.get(u, 1e-6)
    return {k: {"launches": len(v["ids"]), "dram_bytes": v["bytes"], "ms_under_ncu": v["ms"]} for k, v in per.items()}


def main(tag):
    out = ["# ncu summaries, round %s (`--clock-control none`)" % tag, ""]
    os.makedirs(os.path.join(ROOT, "profiles"), exist_ok=True)
    lp = os.path.join(ROOT, "gpurun_out", "%s_launches.csv" % tag)
    if not os.path.exists(lp):
        lp += ".gz"
    if os.path.exists(lp):
        tot, cnt = launches(lp)
        T = sum(tot.values())
        out += ["## Launch list: `ncu --metrics gpu__time_duration.sum --clock-control none " +
                os.environ.get("NCU_LAUNCH_CMD", "python bench.py --steps 1 --warmup 1 --batch 32 --no-cpu-baseline") + "`", "",
                "Per-launch times under ncu are serialised and cold-cache: read the SHARES. Total %.1f ms over %d launches "
                "(warm-up step + timed step + e2e step + profile passes)." % (T, sum(cnt.values())), "",
                "| kernel | launches | total ms | share |", "|---|---:|---:|---:|"]
        for k, v in sorted(tot.items(), key=lambda x: -x[1])[:18]:
            out.append("| `%s` | %d | %.3f | %.1f %% |" % (k[:70], cnt[k], v, 100 * v / T))
        out.append("")
    for f in sorted(os.listdir(os.path.join(ROOT, "gpurun_out"))):
        if not (f.startswith(tag + "_") and (f.endswith(".ncu-rep") or f.endswith(".raw.csv"))):
            continue
        for d in raw(os.path.join(ROOT, "gpurun_out", f)):
            out += ["## `%s` — %s" % (f, d.get("Kernel Name", ("?", ""))[0][:90]), "", "| metric | value |", "|---|---|"]
            for k in KEYS:
                if k in d:
                    out.append("| %s | %s %s |" % (k, d[k][0], d[k][1]))
            out.append("")
    tp = os.path.join(ROOT, "gpurun_out", "%s_dram_bytes.csv" % tag)
    if os.path.exists(tp):
        import json
        tr = traffic(tp)
        mode, batch = os.environ.get("NCU_MODE", "fast"), int(os.environ.get("NCU_BATCH", "32"))
        meta = {"command": "ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum,gpu__time_duration.sum --clock-control none "
                           "python tools/ncu_target.py %d %s" % (batch, mode), "batch": batch, "mode": mode, "kernels": tr}
        json.dump(meta, open(os.path.join(ROOT, "profiles", "%s_traffic.json" % tag), "w"), indent=1)
        out += ["## DRAM traffic per kernel, one forward+post-proc pass at B=%d (%s mode, one chunk)" % (batch, mode), "",
                "| kernel | launches | DRAM bytes (read+write) | per launch |", "|---|---:|---:|---:|"]
        for k, v in sorted(tr.items(), key=lambda x: -x[1]["dram_bytes"])[:12]:
            out.append("| `%s` | %d | %.3f GB | %.1f MB |" % (k, v["launches"], v["dram_bytes"] / 1e9,
                                                          v["dram_bytes"] / 1e6 / max(1, v["launches"])))
        out.append("")
    path = os.path.join(ROOT, "profiles", "%s_ncu_summary.md" % tag)
    open(path, "w").write("\n".join(out) + "\n")
    print(path)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "r1")
