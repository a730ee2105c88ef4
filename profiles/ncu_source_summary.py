"""ncu --set full --import-source on report -> markdown summary committed under profiles/ (stall picture of ONE kernel launch):
    python profiles/ncu_source_summary.py gpurun_out/X.ncu-rep profiles/X.md ["note"]
Splits the warp-state samples into (a) warps parked at the final barrier / EXIT, (b) mbarrier wait loops (SYNCS TRYWAIT + its
branch), (c) everything else, lists the stall reasons of (c), the instruction mix and IPC, and the hottest instructions."""
import collections
import csv
import io
import subprocess
import sys


def page(rep, name):
    out = subprocess.run(["ncu", "-i", rep, "--page", name, "--csv"], capture_output=True, text=True).stdout
    return list(csv.reader(io.StringIO(out)))


def main():
    rep, dst = sys.argv[1], sys.argv[2]
    note = sys.argv[3] if len(sys.argv) > 3 else ""
    raw = page(rep, "raw")
    h, u, d = raw[0], raw[1], raw[2]
    metric = {x: (d[i], u[i]) for i, x in enumerate(h)}
    want = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread", "sm__cycles_elapsed.max",
            "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_sector_hit_rate.pct",
            "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active",
            "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
            "smsp__issue_active.avg.pct_of_peak_sustained_active", "sm__warps_active.avg.pct_of_peak_sustained_active",
            "dram__throughput.avg.pct_of_peak_sustained_elapsed"]
    src = page(rep, "source")
    kname = src[0][1] if src and len(src[0]) > 1 else "?"
    hdr, data = src[1], src[2:]
    ix = {x: i for i, x in enumerate(hdr)}
    stall_cols = [x for x in hdr if x.startswith("stall_") and "Not Issued" not in x]
    recs = []
    for r in data:
        if len(r) < len(hdr):
            continue
        try:
            n, s = int(r[ix["Instructions Executed"]]), int(r[ix["# Samples"]])
        except ValueError:
            continue
        recs.append((r[ix["Source"]].strip(), n, s, {c: int(r[ix[c]] or 0) for c in stall_cols}))
    tot = sum(x[2] for x in recs) or 1
    n_inst = sum(x[1] for x in recs)
    grp = collections.Counter()
    other_st = collections.Counter()
    ops = collections.Counter()
    for i, (s_, n, s, st) in enumerate(recs):
        op = (s_.split()[1] if s_.startswith("@") else s_.split()[0]).split(".")[0] if s_ else "?"
        ops[op] += n
        near_wait = any("TRYWAIT" in recs[j][0] for j in range(max(0, i - 2), i + 1))
        if "EXIT" in s_:
            grp["parked at the final barrier / EXIT"] += s
        elif "TRYWAIT" in s_ or (s_.startswith("@") and "BRA" in s_ and near_wait) or "YIELD" in s_ or "NANOSLEEP" in s_:
            grp["mbarrier wait loops"] += s
        else:
            grp["everything else (compute, stores)"] += s
            for k, v in st.items():
                other_st[k] += v
    lines = [f"# ncu source-level summary: `{kname[:140]}`", "", f"report: `{rep}` (ncu --set full --clock-control none --import-source on, one launch).  {note}", ""]
    lines += ["| metric | value |", "|---|---|"]
    for k in want:
        if k in metric:
            lines.append(f"| {k} | {metric[k][0]} {metric[k][1]} |")
    cyc = float(metric.get("sm__cycles_elapsed.max", ("0", ""))[0] or 0)
    if cyc:
        sched = 132 * 4   # H100 SXM: 132 SMs x 4 schedulers
        lines.append(f"| warp instructions executed / (cycles x 132 SMs x 4 schedulers) | {n_inst} / {cyc * sched:.0f} = {n_inst / (cyc * sched):.3f} IPC per scheduler |")
    lines += ["", f"Warp-state samples: {tot}", "", "| where | share |", "|---|---|"]
    for k, v in grp.most_common():
        lines.append(f"| {k} | {100 * v / tot:.1f} % |")
    o_tot = sum(other_st.values()) or 1
    lines += ["", "Stall reasons inside \"everything else\":", "", "| reason | share |", "|---|---|"]
    for k, v in other_st.most_common(8):
        lines.append(f"| {k} | {100 * v / o_tot:.1f} % |")
    lines += ["", "Instruction mix (warp instructions):", "", "| opcode | count | share |", "|---|---|---|"]
    for k, v in ops.most_common(16):
        lines.append(f"| {k} | {v} | {100 * v / max(n_inst, 1):.1f} % |")
    lines += ["", "Hottest instructions:", "", "| samples | executed | SASS | top stall reasons |", "|---|---|---|---|"]
    for s_, n, s, st in sorted(recs, key=lambda x: -x[2])[:18]:
        top = ", ".join(f"{k[6:]} {v}" for k, v in sorted(st.items(), key=lambda kv: -kv[1])[:2] if v)
        lines.append(f"| {100 * s / tot:.1f} % | {n} | `{s_[:70]}` | {top} |")
    open(dst, "w").write("\n".join(lines) + "\n")
    import json
    json.dump({"kernel": kname[:200], "report": rep, "note": note, "metrics": {k: {"value": metric[k][0], "unit": metric[k][1]} for k in want if k in metric},
               "warp_instructions": n_inst, "sample_groups": {k: v / tot for k, v in grp.items()}}, open(dst.rsplit(".", 1)[0] + ".json", "w"), indent=1)
    print("\n".join(lines[:30]))


if __name__ == "__main__":
    main()
