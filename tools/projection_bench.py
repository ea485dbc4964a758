"""Projection queries over bench.py's c2 table (1e9 HBM-resident rows by default).

    python tools/projection_bench.py [--rows 1e9] [--runs 3] [--json PATH]

Workloads, all `SELECT g, c1 FROM t WHERE c0 < k` with columnar output (c0 uniform in [0, 1e6)):
  sweep      k for ~1 %, 10 %, 50 %, 100 % selectivity, once with result_on_device and once with the default host copy (the host
             copy is skipped when the result exceeds HOST_COPY_MAX_BYTES of pinned memory)
  limit      the 50 % query with LIMIT 1000: kernel time and the rows of the chunks the kernel loaded (B2Q_STAT_ROWS_SCANNED)
  topk       the 50 % query with ORDER BY c1 DESC LIMIT 10
Reported per workload: the projection kernel's CUDA-event time inside libb2q, the step time (host wall-clock of
executeWorkUnit, which includes the COUNT(*) pre-flight of a unit without a scan limit, the sort and the copy back), and the
bytes model below over kernel time, against the H100 SXM data-sheet bandwidth and tools/stream_read.cu's measured ceiling.
Mean of the runs and max - min.  Every run checks the row count against the exact count of passing rows.

Bytes model of one projection kernel: the filter column (8 B per row scanned), plus every 32-byte sector of a projected column
that holds at least one passing row (expected value for uniformly spread passing rows: 1 - (1 - p)^(32 / width)), plus the
output written (8-byte offset word + 4 + 8 bytes per row).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (the c2 table definition and generator; bench.py itself is not run)

DATASHEET_TBS = 3.35
READ_CEILING_TBS = 3.05        # tools/stream_read.cu on the H100 SXM used for the numbers in README.md / DESIGN.md
HOST_COPY_MAX_BYTES = 12 << 30
SPAN = 10**6                   # c0 is uniform in [0, SPAN)


def card():
    import torch
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return torch.cuda.get_device_name(), out


def bytes_model(rows_scanned, p, rows_out):
    sectors = lambda w: rows_scanned * w / 32 * (1 - (1 - p) ** (32 / w))   # noqa: E731
    return int(8 * rows_scanned + 32 * (sectors(4) + sectors(8)) + rows_out * (8 + 4 + 8))


def stat(xs):
    return {"mean": float(np.mean(xs)), "spread": float(np.max(xs) - np.min(xs))}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("projection_bench needs a CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(0)
    from heavydb_b200 import abi, executor, sqlmini
    rows = int(args.rows)
    name, power = card()
    cols = bench.CONFIGS["c2"][0]
    names = [c[0] for c in cols]
    table, keep = bench.build_device_table("c2", bench.rank_fragments(rows, 0, 1), torch)
    ex = executor.Executor()
    eo = executor.execution_options(output_columnar_hint=True)
    # exact passing counts for the checks: one COUNT(*) per threshold through the aggregate path
    def count(k):
        u = sqlmini.parse(f"SELECT COUNT(*) FROM t WHERE c0 < {k}", table, names, bigint_count=True)
        return ex.executeWorkUnit(0, True, table, u, memory_level=abi.GPU_LEVEL).rows()[0][0]

    def run(sql, on_device, expect_rows):
        unit = sqlmini.parse(sql, table, names)
        ex.executeWorkUnit(0, False, table, unit, eo=eo, memory_level=abi.GPU_LEVEL, result_on_device=on_device)   # warm-up
        ks, ss, scanned = [], [], []
        for _ in range(args.runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rs = ex.executeWorkUnit(0, False, table, unit, eo=eo, memory_level=abi.GPU_LEVEL, result_on_device=on_device)
            ss.append((time.perf_counter() - t0) * 1e3)
            ks.append(rs.kernel_ms())
            scanned.append(rs.stats()["rows_scanned"])
            assert rs.rowCount() == expect_rows, (sql, rs.rowCount(), expect_rows)
            del rs
        return {"sql": sql, "result_on_device": on_device, "rows_out": expect_rows, "kernel_ms": stat(ks), "step_ms": stat(ss),
                "rows_scanned": int(np.max(scanned))}

    out = {"card": name, "power_limit": power, "rows": rows, "runs": args.runs, "datasheet_tbs": DATASHEET_TBS,
           "read_ceiling_tbs": READ_CEILING_TBS, "sweep": [], "limit": None, "topk": None}
    for k in (10_000, 100_000, 500_000, 1_000_000):
        p = k / SPAN
        n = count(k)
        for on_device in (True, False):
            if not on_device and n * 20 > HOST_COPY_MAX_BYTES:
                continue
            r = run(f"SELECT g, c1 FROM t WHERE c0 < {k}", on_device, n)
            r["selectivity"] = p
            r["model_bytes"] = bytes_model(rows, p, n)
            tbs = r["model_bytes"] / (r["kernel_ms"]["mean"] / 1e3) / 1e12
            r["model_tbs"], r["of_datasheet"], r["of_read_ceiling"] = tbs, tbs / DATASHEET_TBS, tbs / READ_CEILING_TBS
            print(json.dumps(r), flush=True)
            out["sweep"].append(r)
    out["limit"] = run("SELECT g, c1 FROM t WHERE c0 < 500000 LIMIT 1000", False, 1000)
    print(json.dumps(out["limit"]), flush=True)
    out["topk"] = run("SELECT g, c1 FROM t WHERE c0 < 500000 ORDER BY c1 DESC LIMIT 10", False, 10)
    print(json.dumps(out["topk"]), flush=True)
    del keep, table
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
