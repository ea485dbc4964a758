"""Cost of an IN list planned as a set term (a device bitmap over [min, max] of its values) on 1e9 HBM-resident rows of the c2
shape: SELECT g, SUM(c1), COUNT(*) FROM t WHERE c0 IN (...) OR c0 < 500000 GROUP BY g.

    python tools/in_list_bench.py [--rows 1e9] [--reps 5] [--out FILE]

c0 is uniform in [0, 1e6), so a list alone selects at most its length / 1e6 of the rows; `OR c0 < 500000` brings every query
to about 50 % selectivity with the set term evaluated on every row.  The list values lie at or above 500000, so the baseline
`c0 < 500000 + hits` (one range leaf) selects the same number of rows in expectation.  Lists: 17 values (4 KB bitmap), 1 000 and 100 000 values
over [500000, 1e6) (62.5 KB bitmaps), and 100 000 values spread over 2^30 (a 128 MB bitmap; the rows only reach its first
62.5 KB, so it measures the build and the memory, not a bitmap larger than the caches).  Each list query alternates with the
baseline in one process, --reps timed runs each after two warm-ups.

Reported per query: kernel_ms (the scan's CUDA events, rs.kernel_ms()), build_ms (b2q_k_set_build's device time from
torch.profiler, in a separate profiled run), step_ms (host wall time of executeWorkUnit, which ends in a synchronize), and the
same for the baseline.  Every timed result is checked against an exact numpy group-by of the generated columns.  The card's
name and power limit are read in the same run.  Tables are generated in HBM by bench.py's generator (a ring of 4 resident
32 Mi-row fragments).
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from heavydb_b200 import abi, executor, sqlmini  # noqa: E402
from interrupt_bench import card  # noqa: E402


def lists(rng):
    """name -> sorted list values (all >= 500000)."""
    half = 500_000
    return {
        "17_values_4KB": sorted(rng.sample(range(half, half + 32_768, 2), 17)),
        "1000_values_62KB": sorted(rng.sample(range(half, 10**6, 2), 1000)),
        "100000_values_62KB": sorted(rng.sample(range(half, 10**6, 2), 100_000)),
        "100000_values_128MB": sorted(set([half] + rng.sample(range(half + 2, half + (1 << 30), 2), 99_999))),
    }


class Exact:
    """Exact group-by of the generated table from the 4 physical fragments copied back to the host: per physical fragment,
    the (count, sum) per group of its first m rows for every logical fragment length m that aliases it."""
    def __init__(self, frags, keep):
        self.frags = frags
        self.phys = {}
        k = 0
        for _fid, m, alias in frags:
            if alias not in self.phys:
                c0, c1, g = (keep[k + i].cpu().numpy() for i in range(3))
                k += 3
                self.phys[alias] = (c0.view(np.int64), c1.view(np.int64), g.view(np.int32))

    def groupby(self, mask_of):
        cnt = np.zeros(10**4, np.int64)
        sm = np.zeros(10**4, np.uint64)
        cache = {}
        for _fid, m, alias in self.frags:
            key = (alias, m)
            if key not in cache:
                c0, c1, g = (a[:m] for a in self.phys[alias])
                sel = mask_of(c0)
                gs, vs = g[sel], c1[sel]
                c = np.bincount(gs, minlength=10**4).astype(np.int64)
                order = np.argsort(gs, kind="stable")
                csum = np.concatenate([np.zeros(1, np.uint64), np.cumsum(vs[order].view(np.uint64), dtype=np.uint64)])
                b = np.searchsorted(gs[order], np.arange(10**4 + 1))
                cache[key] = (c, csum[b[1:]] - csum[b[:-1]])
            cnt += cache[key][0]
            sm += cache[key][1]
        return {g: (int(sm[g].astype(np.int64)), int(cnt[g])) for g in np.nonzero(cnt)[0]}


def check(rs, want):
    got = {int(r[0]): (int(r[1]), int(r[2])) for r in rs.rows()}
    assert got == want, "result differs from the exact group-by"


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    rows = int(args.rows)
    frags = bench.rank_fragments(rows, 0, 1, ring=4)
    table, keep = bench.build_device_table("c2", frags, torch)
    names = [c[0] for c in bench.CONFIGS["c2"][0]]
    bt = table.build(abi.GPU_LEVEL)
    exact = Exact(frags, keep)
    ex = executor.Executor()
    result = {"card": card(), "rows": rows, "query": "SELECT g, SUM(c1), COUNT(*) FROM t WHERE c0 IN (...) OR c0 < 500000 GROUP BY g",
              "lists": {}}
    for name, vals in lists(random.Random(1)).items():
        hits = sum(1 for v in vals if v < 10**6)
        sql = f"SELECT g, SUM(c1), COUNT(*) FROM t WHERE c0 IN ({', '.join(map(str, vals))}) OR c0 < 500000 GROUP BY g;"
        base_sql = f"SELECT g, SUM(c1), COUNT(*) FROM t WHERE c0 < {500_000 + hits} GROUP BY g;"
        unit, base = sqlmini.parse(sql, table, names), sqlmini.parse(base_sql, table, names)
        varr = np.array(vals, dtype=np.int64)
        want = exact.groupby(lambda c0: (c0 < 500_000) | np.isin(c0, varr))
        want_base = exact.groupby(lambda c0: c0 < 500_000 + hits)

        def run(u):
            t0 = time.perf_counter()
            rs = ex.executeWorkUnit(0, True, bt, u, memory_level=abi.GPU_LEVEL)
            return rs, (time.perf_counter() - t0) * 1e3
        for _ in range(2):
            run(unit), run(base)
        k, s, kb, sb = [], [], [], []
        for _ in range(args.reps):
            rs, ms = run(unit)
            check(rs, want)
            k.append(rs.kernel_ms()), s.append(ms)
            assert rs.getQueryMemDesc().kernel == abi.KERNEL_PERFECT_SMEM
            launches = rs.stats()["kernel_launches"]
            rb, msb = run(base)
            check(rb, want_base)
            kb.append(rb.kernel_ms()), sb.append(msb)
            assert launches == rb.stats()["kernel_launches"] + 1
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            run(unit)
            torch.cuda.synchronize()
        build_us = sum(e.device_time_total for e in prof.key_averages() if "set_build" in e.key)
        med = statistics.median
        result["lists"][name] = {
            "values": len(vals), "bitmap_bytes": ((vals[-1] - vals[0]) // 32 + 1) * 4, "rows_selected": sum(c for _, c in want.values()),
            "base_rows_selected": sum(c for _, c in want_base.values()),
            "kernel_ms": round(med(k), 3), "base_kernel_ms": round(med(kb), 3), "kernel_vs_base_pct": round(100 * (med(k) - med(kb)) / med(kb), 1),
            "build_ms": round(build_us / 1e3, 3), "step_ms": round(med(s), 2), "base_step_ms": round(med(sb), 2),
            "kernel_all": [round(x, 3) for x in k], "base_kernel_all": [round(x, 3) for x in kb]}
        print(name, result["lists"][name], flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
