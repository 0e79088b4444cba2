"""Turn an `ncu --csv --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum` launch list into
profiles/<tag>_launch_shares.txt and profiles/traffic_by_family.json (average DRAM bytes per launch of the kernels behind
each bench.py family; bench.py reports it as roofline.traffic).

Usage: python tools/ncu_summarise.py gpurun_out/launches.csv r01 "command line that was profiled"
"""
import collections
import csv
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAMILY_KERNELS = {          # bench.py family -> kernels that implement it (the TMA kernel serves fwd and dgrad alike)
    "conv_wgrad_tc": ["conv_wgrad_tc_kernel", "conv_wgrad_thin_kernel"],
    "conv_fwd_tc": ["conv_tma_kernel", "conv_fwd_tc_kernel"],
    "conv_dgrad_tc": ["conv_tma_kernel", "conv_fwd_tc_kernel"],
    "bn_bwd": ["bn_bwd_reduce_kernel", "bn_bwd_apply_kernel", "bn_param_grad_kernel"],
    "bn_apply": ["bn_apply_kernel"],
    "pair_fwd": ["pairwise_fwd_kernel"],
    "pair_bwd": ["pairwise_bwd_kernel"],
}


def to_bytes(v, unit):
    v = float(v.replace(",", ""))
    return v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)


def to_us(v, unit):
    v = float(v.replace(",", ""))
    return v * {"ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6, "nsecond": 1e-3, "usecond": 1, "msecond": 1e3, "second": 1e6}.get(unit, 1)


def main():
    path, tag, cmd = sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else ""
    lines = [l for l in open(path, errors="replace") if l.startswith('"')]
    rows = list(csv.reader(lines))
    hdr = rows[0]
    iid, iname, imet, iunit, ival = (hdr.index(k) for k in ("ID", "Kernel Name", "Metric Name", "Metric Unit", "Metric Value"))
    launches = collections.OrderedDict()
    for r in rows[1:]:
        if len(r) <= ival:
            continue
        d = launches.setdefault(r[iid], {"name": r[iname]})
        if r[imet] == "gpu__time_duration.sum":
            d["us"] = to_us(r[ival], r[iunit])
        elif r[imet] == "dram__bytes_read.sum":
            d["rd"] = to_bytes(r[ival], r[iunit])
        elif r[imet] == "dram__bytes_write.sum":
            d["wr"] = to_bytes(r[ival], r[iunit])
    agg = collections.defaultdict(lambda: [0, 0.0, 0.0, 0.0])
    for d in launches.values():
        name = re.sub(r"^void\s+", "", d["name"])
        name = re.sub(r"^scsfm::", "", name).split("(")[0]
        a = agg[name]
        a[0] += 1
        a[1] += d.get("us", 0.0)
        a[2] += d.get("rd", 0.0)
        a[3] += d.get("wr", 0.0)
    total = sum(a[1] for a in agg.values())
    out = ["# round %s -- ncu launch list of `%s`" % (tag, cmd),
           "# ncu --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum --clock-control none "
           "(cold-cache, serialised: compare SHARES, not absolutes)",
           "# %d launches captured, total %.3f ms" % (len(launches), total / 1e3), "",
           "%-62s %6s %10s %7s %12s %12s" % ("kernel", "count", "total_us", "share", "dram_rd/launch", "dram_wr/launch")]
    for name, a in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        out.append("%-62s %6d %10.1f %6.1f%% %11.2f MB %11.2f MB" % (name[:62], a[0], a[1], 100 * a[1] / total, a[2] / a[0] / 1e6, a[3] / a[0] / 1e6))
    open(os.path.join(ROOT, "profiles", "%s_launch_shares.txt" % tag), "w").write("\n".join(out) + "\n")
    traffic = {}
    for fam, kernels in FAMILY_KERNELS.items():
        n = sum(a[0] for k, a in agg.items() if any(k.startswith(x) for x in kernels))
        b = sum(a[2] + a[3] for k, a in agg.items() if any(k.startswith(x) for x in kernels))
        if n:
            traffic[fam] = {"dram_bytes_per_launch": round(b / n), "launches": n, "kernels": kernels}
    traffic["_source"] = "profiles/%s_launch_shares.txt (ncu, %s)" % (tag, cmd)
    json.dump(traffic, open(os.path.join(ROOT, "profiles", "traffic_by_family.json"), "w"), indent=1)
    print("\n".join(out[:30]))


if __name__ == "__main__":
    main()
