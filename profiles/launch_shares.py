"""ncu launch list (gpu__time_duration.sum per launch, one profiled bench step with a few EAGER decode steps) -> shares of the step
with the decode-step kernels weighted to the 127 steps of the real workload (VERDICT r01: the raw list under-weights decode ~40 x).
    python profiles/launch_shares.py launches.csv launch_shares.md"""
import collections
import csv
import re
import sys

DECODE = re.compile(r"gemm_kernel<(\(int\))?32,|decode_attn_kernel|rmsnorm_rowblock_kernel|rope_table_kernel|argmax_(partial|final)_kernel")
NEW_TOKENS = 128


def main():
    src, dst = sys.argv[1], sys.argv[2]
    rows = list(csv.reader(open(src)))
    hi = [i for i, r in enumerate(rows) if r and r[0] == "ID"][0]
    hdr, data = rows[hi], rows[hi + 1:]
    ki, vi, ui = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = collections.OrderedDict()
    n_steps = 0
    for r in data:
        if len(r) <= vi:
            continue
        v = float(r[vi].replace(",", ""))
        v = v / 1e3 if r[ui] in ("ns", "nsecond") else v * 1e3 if r[ui] in ("ms", "msecond") else v   # -> us
        full = r[ki]
        name = re.sub(r"\(CUtensorMap.*", "", full)[:90]
        dec = bool(DECODE.search(full))
        if "rope_table_kernel" in full:
            n_steps += 1
        a = agg.setdefault(name, [0, 0.0, dec])
        a[0] += 1
        a[1] += v
    w = (NEW_TOKENS - 1) / max(n_steps, 1)
    tot_raw = sum(v[1] for v in agg.values())
    tot_w = sum(v[1] * (w if v[2] else 1.0) for v in agg.values())
    lines = [f"# {src}: ncu --metrics gpu__time_duration.sum --clock-control none, one profiled step; {sum(v[0] for v in agg.values())} launches, "
             f"{tot_raw / 1e3:.1f} ms as profiled, {n_steps} eager decode steps in the profile",
             f"# decode-step kernels (few-token GEMMs, decode attention, row-block RMSNorm, rope table, argmax) weighted x {w:.1f} to the 127 cached steps "
             f"of the workload -> {tot_w / 1e3:.1f} ms; cold-cache serialised launches: compare SHARES with bench.py's stage split, not absolutes",
             "", "| ms weighted | share | launches profiled | decode-step kernel | kernel |", "|---|---|---|---|---|"]
    for k, v in sorted(agg.items(), key=lambda kv: -(kv[1][1] * (w if kv[1][2] else 1.0))):
        ms = v[1] * (w if v[2] else 1.0) / 1e3
        lines.append(f"| {ms:.2f} | {100 * ms * 1e3 / tot_w:.1f} % | {v[0]} | {'yes' if v[2] else ''} | `{k}` |")
    open(dst, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines[:14]))


if __name__ == "__main__":
    main()
