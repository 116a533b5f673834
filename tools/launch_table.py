"""Turn an ncu launch list (`--metrics gpu__time_duration.sum,launch__grid_size,dram__bytes_read.sum,dram__bytes_write.sum
--csv`) of `bench.py --graph 0` into (1) a per-kernel summary of ONE step and (2) the table of that step's wgmma NT
launches (epilogue, grid, duration, DRAM bytes).  Usage: python tools/launch_table.py launches.csv [launches_per_step]"""
import collections
import csv
import re
import sys


def load(path):
    lines = [l for l in open(path) if not l.startswith("==")]
    byid = collections.OrderedDict()
    for r in csv.DictReader(lines):
        d = byid.setdefault(r["ID"], {"name": r["Kernel Name"]})
        v = float(r["Metric Value"].replace(",", ""))
        u = r["Metric Unit"]
        if r["Metric Name"] == "gpu__time_duration.sum":
            v = v / 1e3 if u in ("nsecond", "ns") else (v * 1e3 if u in ("msecond", "ms") else v)
        if "bytes" in r["Metric Name"]:
            v = v * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
        d[r["Metric Name"]] = v
    return list(byid.values())


def short(n):
    m = re.search(r"(Epi\w+)", n)
    k = re.sub(r"^void\s+", "", n).replace("(anonymous namespace)::", "").replace("<unnamed>::", "")
    mm = re.match(r"[A-Za-z_][A-Za-z0-9_:]*", k)
    k = mm.group(0) if mm else n[:30]
    return k + ("<" + m.group(1) + ">" if m and "gemm" in k else "")


def main():
    L = load(sys.argv[1])
    per_step = int(sys.argv[2]) if len(sys.argv) > 2 else None
    idx = [i for i, d in enumerate(L) if "k_pack_linear" in d["name"]]      # first kernel of a step
    a = idx[0] if idx else 0
    W = L[a:] + L[:a]
    if per_step:
        W = W[:per_step]
    tot = collections.defaultdict(lambda: [0, 0.0])
    for d in W:
        tot[short(d["name"])][0] += 1
        tot[short(d["name"])][1] += d["gpu__time_duration.sum"]
    T = sum(v[1] for v in tot.values())
    print(f"one step = {len(W)} launches, sum of per-launch durations {T:.1f} us (ncu: serialised, cold cache, no PDL overlap)")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1][1])[:50]:
        print(f"{v[1]:9.1f} us {100 * v[1] / T:5.1f}% n={v[0]:3d} avg {v[1] / v[0]:7.1f}  {k}")
    print()
    print("fused value-chain launches of the step (k_sdf_chain): grid, us, DRAM MB (read+write)")
    for d in W:
        if "k_sdf_chain" in d["name"]:
            mb = (d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)) / 1e6
            print(f"  k_sdf_chain    grid {int(d.get('launch__grid_size', 0)):4d} {d['gpu__time_duration.sum']:7.1f} us {mb:7.1f} MB")
    print()
    print("wgmma NT launches of the step, in launch order: epilogue, grid, us, DRAM MB (read+write), GB/s")
    for d in W:
        if "gemm_tc_nt" in d["name"]:
            mb = (d.get("dram__bytes_read.sum", 0.0) + d.get("dram__bytes_write.sum", 0.0)) / 1e6
            us = d["gpu__time_duration.sum"]
            print(f"  {short(d['name']).split('<')[1][:-1]:14s} grid {int(d.get('launch__grid_size', 0)):4d} {us:7.1f} us "
                  f"{mb:7.1f} MB {mb / us * 1e3 if us else 0:7.0f} GB/s")


if __name__ == "__main__":
    main()
