#!/usr/bin/env python
"""Per-kernel totals and shares of an `ncu --metrics gpu__time_duration.sum --csv` launch list (cold-cache, serialised
launches: compare SHARES with the in-graph ablation, never the absolute times).

  python tools/launch_shares.py launches.csv [--top 20]
"""
import argparse
import collections
import csv
import json


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--top", type=int, default=20)
    a = ap.parse_args()
    rows = list(csv.reader(open(a.csv)))
    hi = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    hdr = rows[hi]
    kn, mv, mu = hdr.index("Kernel Name"), hdr.index("Metric Value"), hdr.index("Metric Unit")
    agg = collections.defaultdict(lambda: [0, 0.0])
    for r in rows[hi + 1:]:
        if len(r) <= mv:
            continue
        v = float(r[mv].replace(",", ""))
        if r[mu] == "ns":
            v /= 1e3
        name = r[kn].split("(")[0].replace("void ", "")
        agg[name][0] += 1
        agg[name][1] += v
    tot = sum(v for _, v in agg.values())
    ours = sum(v for k, (_, v) in agg.items() if k.startswith("lade::"))
    lib = sum(v for k, (_, v) in agg.items() if k.startswith("nvjet"))
    print(json.dumps({"launches": sum(n for n, _ in agg.values()), "total_us": round(tot, 1),
                      "share_own_kernels_pct": round(100 * ours / tot, 1), "share_cublas_nvjet_pct": round(100 * lib / tot, 1)}))
    for k, (n, v) in sorted(agg.items(), key=lambda kv: -kv[1][1])[: a.top]:
        print(f"{k[:72]:72s} n={n:5d} total={v:10.1f} us  mean={v / n:8.2f}  share={100 * v / tot:5.1f}%")


if __name__ == "__main__":
    main()
