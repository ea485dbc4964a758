"""Temporary tables: what the chunk stats cost the conversion kernel, and how long the hand-off to a second step takes.

    python tools/temp_table_bench.py [--rows 1e9] [--configs c2,c4,c4s] [--runs 3] [--parent-tree DIR] [--json PATH]

The tables and step-1 queries are bench.py's c2 / c4 / c4s (same generator, seed, fragment size, in HBM); step 1 also counts
its groups, as the reference's Aggregate does for a HAVING COUNT(*) (sqlmini.parse_steps).  Step 2 reads step 1's result as
a temporary table:

    SELECT COUNT(*), SUM(s) FROM (SELECT <key>, SUM(<v>) AS s, COUNT(*) AS n FROM t GROUP BY <key>) WHERE n > k

with k the median group count (about 50 % of the groups pass).  Reported per config, mean and max - min of --runs runs:

  1. convert_kernel_ms: b2q_device_columns_convert_ms of step 1's result, this tree against --parent-tree (a copy of the
     parent commit with its library built, e.g. `git archive <parent> | tar -x -C DIR` then `python -m heavydb_b200.build`
     there).  The two trees run in alternating worker processes in one session.
  2. handoff_ms: host wall-clock from step 1's return to step 2's result.
       device route  b2q_rs_device_columns (columns + chunk stats) -> as_table() -> step 2 on the GPU_LEVEL table
       host route    the reference's: b2q_columnar_results_create + synthesize_metadata on the host (numpy restatement,
                     tests/temp_table_ref.py) -> step 2 on a CPU_LEVEL table (the H2D copy happens inside that call)
     Step 1 runs with result_on_device for the device route and without it for the host route.  Every run checks that
     both routes return the same step-2 row.
The card name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    import torch
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def step1_sql(cfg):
    import bench
    cols = bench.CONFIGS[cfg][0]
    sql = bench.CONFIGS[cfg][1]
    return (sql if "COUNT(*)" in sql else sql.replace(" FROM t", ", COUNT(*) FROM t")), cols


def worker(tree, configs, rows, reps):
    """Conversion-kernel time of step 1's result, with the heavydb_b200 package (and its library) of `tree`."""
    sys.path[:0] = [tree, os.path.join(tree, "tests")]
    import torch
    import bench
    from heavydb_b200 import abi, executor, sqlmini
    torch.cuda.set_device(0)
    out = {}
    for cfg in configs:
        sql, cols = step1_sql(cfg)
        names = [c[0] for c in cols]
        table, keep = bench.build_device_table(cfg, bench.rank_fragments(rows, 0, 1), torch)
        unit = sqlmini.parse(sql, table, names)
        guess = bench.ENTRY_GUESS.get(cfg, 0)
        ex = executor.Executor()
        ms = []
        for r in range(reps + 1):
            rs = ex.executeWorkUnit(guess, True, table, unit, has_cardinality_estimation=guess > 0, memory_level=abi.GPU_LEVEL,
                                    result_on_device=True)
            dc = rs.deviceColumns(stream=0)
            if r:             # the first conversion is a warm-up
                ms.append(dc.convert_ms())
            del dc, rs
        out[cfg] = float(np.mean(ms))
        del keep, table
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


def convert_comparison(parent, configs, rows, runs, reps):
    res = {cfg: {"this": [], "parent": []} for cfg in configs}
    for _ in range(runs):
        for arm, tree in (("parent", parent), ("this", ROOT)):
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, "--configs", ",".join(configs),
                                "--rows", str(rows), "--reps", str(reps)], capture_output=True, text=True, check=True)
            for cfg, ms in json.loads(p.stdout.strip().splitlines()[-1]).items():
                res[cfg][arm].append(ms)
    return res


def handoff(cfg, rows, runs, torch):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import bench
    import temp_table_ref as tt
    from heavydb_b200 import abi, executor, sqlmini
    _sql1, cols = step1_sql(cfg)
    key, val = ("g", "c1") if cfg.startswith("c2") else (cols[0][0], cols[1][0])
    names = [c[0] for c in cols]
    table, keep = bench.build_device_table(cfg, bench.rank_fragments(rows, 0, 1), torch)
    guess = bench.ENTRY_GUESS.get(cfg, 0)
    ex = executor.Executor()
    kw1 = dict(has_cardinality_estimation=guess > 0, memory_level=abi.GPU_LEVEL)
    inner = f"SELECT {key}, SUM({val}) AS s, COUNT(*) AS n FROM t GROUP BY {key}"
    if cfg.startswith("c2"):
        inner = f"SELECT {key}, SUM({val}) AS s, COUNT(*) AS n FROM t WHERE c0 < 500000 GROUP BY {key}"
    probe = sqlmini.parse_steps(f"SELECT COUNT(*) FROM ({inner});", table, names)
    unit1 = sqlmini.parse(probe[0].sql, table, names)
    # k: the median group count
    rs = ex.executeWorkUnit(guess, True, table, unit1, result_on_device=True, **kw1)
    dc = rs.deviceColumns(stream=0)
    n_col = dc.tensors()[2][0]
    k = int(torch.median(n_col.to(torch.int64)).item())
    del dc, rs
    steps = sqlmini.parse_steps(f"SELECT COUNT(*), SUM(s) FROM ({inner}) WHERE n > {k};", table, names)
    assert len(steps) == 2
    out = {"device_ms": [], "host_ms": [], "convert_ms": [], "rows_step1": None, "k": k, "sql": steps[1].sql}
    for r in range(runs + 1):
        # device route
        rs1 = ex.executeWorkUnit(guess, True, table, unit1, result_on_device=True, **kw1)
        t0 = time.perf_counter()
        dc = rs1.deviceColumns(stream=0)
        tmp = dc.as_table()
        unit2 = sqlmini.parse(steps[1].sql, tmp, steps[0].names)
        rs2 = ex.executeWorkUnit(0, True, tmp, unit2, memory_level=abi.GPU_LEVEL)
        dev_row = rs2.rows()
        t1 = time.perf_counter()
        assert rs1.stats()["result_d2h_bytes"] == 0
        convert = dc.convert_ms()
        n1 = dc.size()
        del rs2, tmp, dc, rs1
        # host route
        rs1 = ex.executeWorkUnit(guess, True, table, unit1, **kw1)
        t2 = time.perf_counter()
        host_cols = rs1.columnarResults(num_threads=os.cpu_count() or 1, with_scale=True)
        htmp = tt.host_table(host_cols)
        hunit2 = sqlmini.parse(steps[1].sql, htmp, steps[0].names)
        rs2 = ex.executeWorkUnit(0, True, htmp, hunit2, memory_level=abi.CPU_LEVEL)
        host_row = rs2.rows()
        t3 = time.perf_counter()
        assert dev_row == host_row, (dev_row, host_row)
        del rs2, htmp, host_cols, rs1
        if r:     # the first run is a warm-up
            out["device_ms"].append((t1 - t0) * 1e3)
            out["host_ms"].append((t3 - t2) * 1e3)
            out["convert_ms"].append(convert)
            out["rows_step1"] = n1
            out["step2_row"] = [list(x) for x in dev_row]
    del keep, table
    torch.cuda.empty_cache()
    return out


def stat(xs):
    return {"mean": float(np.mean(xs)), "spread": float(np.max(xs) - np.min(xs)), "runs": [float(x) for x in xs]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--configs", default="c2,c4,c4s")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=5, help="conversions per worker run (mean taken)")
    ap.add_argument("--parent-tree", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    configs = args.configs.split(",")
    if args.worker:
        worker(args.worker, configs, int(args.rows), args.reps)
        return
    import torch
    if not torch.cuda.is_available():
        sys.exit("temp_table_bench needs a CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(0)
    name, power = card()
    out = {"card": name, "power_limit": power, "rows": int(args.rows), "runs": args.runs, "configs": {}}
    if args.parent_tree:
        conv = convert_comparison(os.path.abspath(args.parent_tree), configs, int(args.rows), args.runs, args.reps)
        for cfg in configs:
            out["configs"].setdefault(cfg, {})["convert_kernel_ms"] = {arm: stat(v) for arm, v in conv[cfg].items()}
        print(json.dumps({"convert_kernel_ms": out["configs"]}), flush=True)
    for cfg in configs:
        h = handoff(cfg, int(args.rows), args.runs, torch)
        out["configs"].setdefault(cfg, {})["handoff_ms"] = {"device_route": stat(h["device_ms"]), "host_route": stat(h["host_ms"]),
                                                           "convert_ms_in_device_route": stat(h["convert_ms"]),
                                                           "rows_step1": h["rows_step1"], "k": h["k"], "step2_sql": h["sql"],
                                                           "step2_row": h["step2_row"]}
        print(json.dumps({cfg: out["configs"][cfg]}), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
