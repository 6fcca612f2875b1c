"""Turn gpurun_out/r01_*.ncu-rep + r01_launches.csv into the small text/JSON summaries that are
committed under profiles/ (the .ncu-rep files themselves stay in gpurun_out/, scratch)."""
import collections
import csv
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "gpurun_out")
DST = os.path.join(ROOT, "profiles")
TAG = sys.argv[1] if len(sys.argv) > 1 else "r01"

KEEP = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts.sum.pct_of_peak_sustained_elapsed",
    "l1tex__m_l1tex2xbar_req_cycles_active.avg.pct_of_peak_sustained_elapsed",
    "l1tex__m_xbar2l1tex_read_bytes.sum", "l1tex__m_l1tex2xbar_write_bytes.sum",
    "sm__throughput.avg.pct_of_peak_sustained_elapsed", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread", "launch__grid_size",
    "launch__block_size", "smsp__inst_executed.sum", "smsp__thread_inst_executed_per_inst_executed.ratio",
    "sm__pipe_fp64_cycles_active.avg.pct_of_peak_sustained_active", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "sm__cycles_elapsed.avg.per_second",
]


def raw(rep):
    """-> (header, units, [one row per DISTINCT kernel in the report, first launch of each])."""
    out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(out.splitlines()))
    hdr = rows[0]
    ki = hdr.index("Kernel Name") if "Kernel Name" in hdr else None
    seen, keep = set(), []
    for r in rows[2:]:
        key = r[ki] if ki is not None else len(keep)
        if key not in seen:
            seen.add(key)
            keep.append(r)
    return hdr, rows[1], keep


def short_name(kernel):
    """vidar::<unnamed>::msda_backward_kernel<8, 0>(...) -> msda_backward"""
    k = kernel.split("(")[0].split("::")[-1]
    k = k.split("<")[0]
    return k[:-7] if k.endswith("_kernel") else k


def main():
    os.makedirs(DST, exist_ok=True)
    traffic = {}
    lines = [f"# ncu --set full --clock-control none, first launch of each kernel in one bench.py step ({TAG}; tools/profile_round.sh)", ""]
    for f in sorted(os.listdir(SRC)):
        if not (f.startswith(TAG + "_") and f.endswith(".ncu-rep")):
            continue
        hdr, units, kernels = raw(os.path.join(SRC, f))
        for vals in kernels:
            name = vals[hdr.index("Kernel Name")] if "Kernel Name" in hdr else f
            section = f[len(TAG) + 1:-8] if len(kernels) == 1 else short_name(name)
            lines.append(f"## {section}  ({name[:90]})")
            rec = {}
            for k in KEEP:
                if k in hdr:
                    i = hdr.index(k)
                    lines.append(f"  {k:88s} {vals[i]:>16s} {units[i]}")
                    rec[k] = (vals[i], units[i])
            lines.append("")

            def to_bytes(key):
                v, u = rec.get(key, ("0", "byte"))
                mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
                return float(v.replace(",", "")) * mult
            traffic[section] = to_bytes("dram__bytes_read.sum") + to_bytes("dram__bytes_write.sum")
    with open(os.path.join(DST, f"{TAG}_ncu_summary.txt"), "w") as fh:
        fh.write("\n".join(lines))
    # launch list -> per-kernel totals and shares
    lc = os.path.join(SRC, f"{TAG}_launches.csv")
    if os.path.exists(lc):
        with open(lc) as fh:
            body = [l for l in fh if not l.startswith("==")]
        agg = collections.defaultdict(list)
        for row in csv.DictReader(body):
            try:
                agg[row["Kernel Name"]].append(float(row["Metric Value"]))
            except (KeyError, ValueError):
                pass
        tot = sum(sum(v) for v in agg.values())
        with open(os.path.join(DST, f"{TAG}_launches_summary.txt"), "w") as fh:
            fh.write(f"# ncu --metrics gpu__time_duration.sum --clock-control none, bench.py --steps 2 --warmup 3 ({TAG}); "
                     "cold-cache serialised launches: compare SHARES\n")
            for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
                fh.write(f"{sum(v) / tot * 100:6.2f}%  n={len(v):4d}  total={sum(v) / 1e6:9.3f} ms  avg={sum(v) / len(v) / 1e3:9.1f} us  {k[:110]}\n")
    with open(os.path.join(DST, "roofline_traffic.json"), "w") as fh:
        json.dump({"msda_bwd": traffic.get("msda_backward"), "msda_fwd": traffic.get("msda_forward"),
                   "tag": TAG,
                   "all_dram_bytes_per_launch": traffic, "source": f"profiles/{TAG}_ncu_summary.txt"}, fh, indent=1)
    print(open(os.path.join(DST, f"{TAG}_launches_summary.txt")).read()[:1800])


def sass_evidence(lib="vidar_b200/libvidar_b200.so", out="profiles/r02_sass_evidence.txt"):
    """`cuobjdump -sass` mnemonic counts per kernel -> profiles/ (what proves Hopper-native code:
    HGMMA, REDG...F32x4, UTMALDG / UTMAREDG, SYNCS).  python tools/summarize_profiles.py --sass"""
    import collections
    import re
    import subprocess
    sass = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    cur, stats = None, collections.OrderedDict()
    pat = re.compile(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Za-z0-9_.]+)")
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            stats[cur] = collections.Counter()
            continue
        m = pat.match(line)
        if m and cur:
            stats[cur][m.group(1)] += 1
    keys = ["HGMMA", "RED", "LDG.E.NA", "LDG.E.128", "UTMALDG", "UTMAREDG", "SYNCS", "DFMA", "ATOMS", "SHFL", "BAR"]
    names = subprocess.run(["c++filt"], input="\n".join(stats), capture_output=True, text=True).stdout.splitlines()
    lines = ["SASS evidence for " + lib + " (sm_90a): `cuobjdump -sass` mnemonic counts per kernel (tools/summarize_profiles.py --sass).",
             "HGMMA = wgmma (Hopper tensor cores); RED = red.global.add (the .F32x4 form is the 16-byte vector reduction); LDG.E.NA = "
             "ld.global.nc.L1::no_allocate; UTMALDG / UTMAREDG = cp.async.bulk.tensor / cp.reduce.async.bulk.tensor (TMA); SYNCS = mbarrier.", ""]
    for (mangled, c), d in zip(stats.items(), names):
        short = re.sub(r"\(.*", "", d.replace("vidar::(anonymous namespace)::", ""))
        cells = []
        for k in keys:
            hits = {kk: v for kk, v in c.items() if kk.startswith(k)}
            if hits:
                cells.append(f"{k}:{sum(hits.values())}" + (f"({max(hits, key=hits.get)})" if k == "RED" else ""))
        lines.append(f"{short:72s} instrs {sum(c.values()):6d}  " + "  ".join(cells))
    with open(out, "w") as fh:
        fh.write("\n".join(lines) + "\n")
    return out


if __name__ == "__main__":
    if "--sass" in sys.argv:
        print(sass_evidence())
    else:
        main()
