"""Reduce an ncu launch list (``--metrics gpu__time_duration.sum[,dram__bytes_read.sum,dram__bytes_write.sum] --csv``) of a
bench command to ONE forward: per-kernel share of the step, and the DRAM traffic of the tensor-core kernels.

    python tools/summarize_launches.py <launches.csv> <summary.csv> [<traffic.json>]

One forward = the launches from the LAST ``patchify4_kernel`` (the first kernel of a forward) to the end of the list or the next
one.  Per-launch times under ncu are cold-cache and serialised: only the kernel SHARES compare with bench.py.
"""
import csv
import json
import re
import sys
from collections import OrderedDict


def short(name):
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(.*$", "", name)
    return name.replace("mqdet::", "")


def main():
    src, dst = sys.argv[1], sys.argv[2]
    rows = []
    with open(src, newline="") as f:
        lines = [ln for ln in f if ln.startswith('"')]
    rd = csv.DictReader(lines)
    launches = OrderedDict()
    for r in rd:
        e = launches.setdefault(r["ID"], {"name": r["Kernel Name"]})
        try:
            e[r["Metric Name"]] = float(r["Metric Value"].replace(",", ""))
        except ValueError:
            pass
        e.setdefault("unit_" + r["Metric Name"], r["Metric Unit"])
    ls = list(launches.values())
    starts = [i for i, e in enumerate(ls) if "patchify4_kernel" in e["name"]]
    if not starts:
        raise SystemExit("no patchify4_kernel launch found: cannot delimit a forward")
    # the last COMPLETE forward: between the two last starts if there are several, else from the only start to the end
    a, b = (starts[-2], starts[-1]) if len(starts) >= 2 else (starts[-1], len(ls))
    fw = ls[a:b]

    def ns(e):
        v = e.get("gpu__time_duration.sum", 0.0)
        u = e.get("unit_gpu__time_duration.sum", "ns")
        return v * {"ns": 1.0, "us": 1e3, "ms": 1e6, "s": 1e9}.get(u, 1.0)

    def byts(e, k):
        v = e.get(k, 0.0)
        u = e.get("unit_" + k, "byte")
        return v * {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1.0)

    total = sum(ns(e) for e in fw)
    agg = OrderedDict()
    for e in fw:
        k = short(e["name"])
        g = agg.setdefault(k, [0.0, 0, 0.0])
        g[0] += ns(e)
        g[1] += 1
        g[2] += byts(e, "dram__bytes_read.sum") + byts(e, "dram__bytes_write.sum")
    with open(dst, "w") as f:
        f.write(f"# ncu launch list {src}: one forward of the bench command (B=8), {len(fw)} launches, {total / 1e6:.2f} ms serialised\n")
        f.write("# per-launch times are cold-cache and serialised; kernel SHARES are what compares with bench.py\n")
        f.write("share_pct,ms,launches,dram_MB,kernel\n")
        for k, (t, n, d) in sorted(agg.items(), key=lambda kv: -kv[1][0]):
            f.write(f"{100 * t / total:.1f},{t / 1e6:.3f},{n},{d / 1e6:.1f},{k}\n")
    if len(sys.argv) > 3:
        gem = [e for e in fw if any(k in e["name"] for k in ("gemm_wg_kernel", "dcn_conv_kernel", "biattn_image_kernel", "biattn_text_kernel"))]
        d = sum(byts(e, "dram__bytes_read.sum") + byts(e, "dram__bytes_write.sum") for e in gem)
        json.dump({"kernel": "tensor-core kernels (gemm_wg, dcn_conv, biattn_image, biattn_text: all launches of one forward)", "launches": len(gem),
                   "dram_bytes_per_step": d, "dram_bytes_per_launch": d / max(1, len(gem)),
                   "source": f"ncu --metrics dram__bytes_read.sum,dram__bytes_write.sum over the tensor-core launches of one forward ({src})"},
                  open(sys.argv[3], "w"), indent=1)


if __name__ == "__main__":
    main()
