"""Summaries of ncu outputs as markdown tables (ncu reads the reports without a GPU).
  python tools/summarize_ncu.py launches <launches.csv> <out.md> [title]
  python tools/summarize_ncu.py report <file.ncu-rep> <out.md> [title]
  python tools/summarize_ncu.py table <file.ncu-rep | raw.csv> <out.md> [title]     one row per launch, the columns the round's analysis uses"""
import collections
import csv
import subprocess
import sys


def launches(path, out, title):
    lines = [l for l in open(path) if not l.startswith("==")]
    rows = [(r["Kernel Name"], float(r["Metric Value"].replace(",", "")), r["Grid Size"], r["Block Size"]) for r in csv.DictReader(lines)
            if r.get("Metric Name") == "gpu__time_duration.sum"]
    agg = collections.OrderedDict()
    for k, v, g, b in rows:
        name = k.split("(")[0]
        a = agg.setdefault(name, [0, 0.0, g, b]); a[0] += 1; a[1] += v
    tot = sum(a[1] for a in agg.values())
    with open(out, "w") as f:
        f.write(f"# {title}\n\nSource: `ncu --metrics gpu__time_duration.sum --clock-control none` ({len(rows)} launches; times are cold-cache and "
                "serialised: compare SHARES, not absolutes).\n\n| kernel | launches | total us | avg us | share | grid | block |\n|---|---:|---:|---:|---:|---|---|\n")
        for k, a in sorted(agg.items(), key=lambda x: -x[1][1]):
            f.write(f"| `{k}` | {a[0]} | {a[1] / 1000:.1f} | {a[1] / a[0] / 1000:.2f} | {a[1] / tot * 100:.1f}% | {a[2]} | {a[3]} |\n")
        f.write(f"\ntotal {tot / 1000:.1f} us over {len(rows)} launches\n")


WANT = ["gpu__time_duration.sum", "launch__registers_per_thread", "launch__grid_size", "launch__block_size", "launch__cluster",
        "launch__shared_mem_per_block_dynamic", "sm__warps_active.avg.per_cycle_active", "smsp__inst_executed.sum",
        "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_bytes.sum", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
        "smsp__average_warp_latency_per_inst_issued.ratio", "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
        "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
        "sass__inst_executed_local_loads", "sass__inst_executed_local_stores", "smsp__thread_inst_executed_per_inst_executed.ratio",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "sm__throughput.avg.pct_of_peak_sustained_elapsed"]


def report(path, out, title):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(raw.splitlines()))
    hdr = rows[0]
    with open(out, "w") as f:
        f.write(f"# {title}\n\nSource: `ncu --set full --clock-control none --import-source on`, read with `ncu -i {path.split('/')[-1]} --page raw --csv`.\n")
        for vals in rows[2:]:
            d = dict(zip(hdr, vals))
            f.write(f"\n## {d.get('Kernel Name', '?')[:100]}\n\n| metric | value |\n|---|---:|\n")
            for h, v in zip(hdr, vals):
                if h in WANT or any(h.startswith(w) for w in ("launch__cluster",)):
                    f.write(f"| `{h}` | {v} |\n")


def _num(x):
    try:
        return float(x.replace(",", ""))
    except Exception:  # noqa: BLE001
        return float("nan")


def table(path, out, title):
    if path.endswith(".csv"):
        raw = open(path).read()
    else:
        raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader([l for l in raw.splitlines() if not l.startswith("==")]))
    hdr, units = rows[0], rows[1]
    unit = dict(zip(hdr, units))
    stall_cols = [h for h in hdr if h.startswith("smsp__average_warps_issue_stalled_") and h.endswith("_per_issue_active.ratio")]
    tot_dur = tot_sm = 0.0
    lines = []
    for vals in rows[2:]:
        d = dict(zip(hdr, vals))
        dur = _num(d["gpu__time_duration.sum"]) * (1e-3 if unit.get("gpu__time_duration.sum") == "ns" else 1.0)
        dr, dw = _num(d.get("dram__bytes_read.sum", "nan")), _num(d.get("dram__bytes_write.sum", "nan"))
        scale = {"byte": 1e-3, "Kbyte": 1.0, "Mbyte": 1e3, "Gbyte": 1e6}
        dr *= scale.get(unit.get("dram__bytes_read.sum"), 1.0); dw *= scale.get(unit.get("dram__bytes_write.sum"), 1.0)
        st = sorted(((_num(d[c]), c[len("smsp__average_warps_issue_stalled_"):-len("_per_issue_active.ratio")]) for c in stall_cols if d.get(c)), reverse=True)
        sm_act = _num(d.get("sm__cycles_active.sum", "nan"))
        tot_dur += dur; tot_sm += sm_act if sm_act == sm_act else 0.0
        lines.append("| `%s` | %s | %s | %s | %.1f | %.0f | %.1f | %.1f | %.0f | %.0f | %.0f | %.0f | %s |" % (
            d["Kernel Name"].split("(")[0][-44:], d.get("launch__grid_size", "?"), d.get("launch__block_size", "?"), d.get("launch__registers_per_thread", "?"),
            dur, _num(d["smsp__inst_executed.sum"]) / 1e3, _num(d["smsp__issue_active.avg.pct_of_peak_sustained_active"]),
            _num(d["smsp__thread_inst_executed_per_inst_executed.ratio"]), sm_act / 1e3, dr + dw, _num(d.get("l1tex__t_sector_hit_rate.pct", "nan")),
            _num(d.get("lts__t_sector_hit_rate.pct", "nan")), ", ".join("%s %.1f" % (n, v) for v, n in st[:2])))
    with open(out, "w") as f:
        f.write(f"# {title}\n\nSource: `ncu --set full --clock-control none`, one row per launch in launch order (times are cold-cache and serialised).  "
                "inst = warp instructions executed (thousands); issue = `smsp__issue_active` % of peak; thr/inst = active threads per warp instruction; "
                "SM-act = `sm__cycles_active.sum` (thousand cycles summed over the SMs: what the launch costs a GPU shared with other chains); "
                "DRAM = bytes read + written (KB); stalls = the two largest `warps_issue_stalled_*_per_issue_active` ratios.\n\n"
                "| kernel | grid | block | regs | µs | inst k | issue % | thr/inst | SM-act k | DRAM KB | L1 hit % | L2 hit % | top stalls |\n|---|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---:|---|\n")
        f.write("\n".join(lines))
        f.write(f"\n\ntotal {tot_dur:.1f} µs, {tot_sm / 1e3:.0f} k SM-active cycles over {len(lines)} launches\n")


if __name__ == "__main__":
    mode, path, out = sys.argv[1:4]
    title = sys.argv[4] if len(sys.argv) > 4 else path
    {"launches": launches, "report": report, "table": table}[mode](path, out, title)
