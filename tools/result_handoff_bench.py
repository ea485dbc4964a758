"""Result hand-off: host ColumnarResults after the default call vs device columns after a `result_on_device` call.

    python tools/result_handoff_bench.py [--rows 1e9] [--configs c2,c4,c4s] [--runs 3] [--json PATH]

The tables are bench.py's (same counter-based generator, seed, column tags and fragment size, generated in HBM through
b2q_gen_column); the queries are bench.py's c2 / c4 / c4s.  Per config and run:
  host hand-off    executeWorkUnit (result copied to pinned host memory) + ColumnarResults on the host
  device hand-off  executeWorkUnit(result_on_device) + b2q_rs_device_columns
both as host wall-clock until the columns exist, plus the conversion kernel's CUDA-event time and its bytes read +
written per second.  Every run checks the device columns against the host columns of the same query (integers bit for
bit, floating-point sums within 1e-6 relative).  Reports the mean of the runs and max - min.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402  (the workload definitions; bench.py itself is not run)

READ_CEILING_TBS = 3.05   # tools/stream_read.cu on the H100 SXM used for the numbers in README.md / DESIGN.md


def card():
    import torch
    name = torch.cuda.get_device_name()
    try:
        out = subprocess.run(["nvidia-smi", f"--id={torch.cuda.current_device()}", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        out = "unknown"
    return name, out


def conversion_bytes(plan, n_rows, cols):
    """Bytes the conversion moves: every kept entry's row of the materialised buffer read once (row-wise: the whole row;
    columnar: each slot / key column), every target column and its validity words written once."""
    from heavydb_b200 import abi
    if plan.output_columnar:
        keyed = plan.query_desc_type != abi.NonGroupedAggregate and not plan.keyless_hash
        row = (8 * max(plan.num_group_cols, 1) if keyed else 0) + sum(plan.slot_padded_width[s] for s in range(plan.num_slots))
    else:
        row = plan.row_size
    written = sum(a.itemsize * n_rows + 4 * ((n_rows + 31) // 32) for _, _, a, _, _ in cols)
    return row * n_rows, written


def parity(dev_cols, host_cols, baseline):
    from heavydb_b200 import abi
    assert len(dev_cols) == len(host_cols)
    dev = [a for _, _, a, _, _ in dev_cols]
    host = [a for _, _, a in host_cols]
    if baseline and dev and dev[0].size:   # slot order depends on which thread claimed a slot first: compare by key
        dev = [a[np.argsort(dev[0], kind="stable")] for a in dev]
        host = [a[np.argsort(host[0], kind="stable")] for a in host]
    for (ty, _, _, mask, nulls), a, b in zip(dev_cols, dev, host):
        assert a.dtype == b.dtype and a.size == b.size
        if a.dtype.kind == "f":
            assert np.all((a == b) | (np.abs(a - b) <= 1e-6 * np.abs(b)))
        else:
            assert np.array_equal(a, b)
        sentinel = b == abi.NULL_OF[ty]
        assert nulls == int(sentinel.sum()) and ((mask is None) == (nulls == 0))


def run_config(cfg, rows, runs, torch):
    from heavydb_b200 import abi, executor
    cols, sql = bench.CONFIGS[cfg][0], bench.CONFIGS[cfg][1]
    names = [c[0] for c in cols]
    table, keep = bench.build_device_table(cfg, bench.rank_fragments(rows, 0, 1), torch)
    unit = bench.make_unit(cfg, sql, table, names)
    guess = bench.ENTRY_GUESS.get(cfg, 0)
    ex = executor.Executor()
    kw = dict(has_cardinality_estimation=guess > 0, memory_level=abi.GPU_LEVEL)
    threads = os.cpu_count() or 1

    def host_handoff():
        t0 = time.perf_counter()
        rs = ex.executeWorkUnit(guess, True, table, unit, **kw)
        cr = rs.columnarResults(num_threads=threads)
        return time.perf_counter() - t0, rs, cr

    def device_handoff():
        t0 = time.perf_counter()
        rs = ex.executeWorkUnit(guess, True, table, unit, result_on_device=True, **kw)
        t1 = time.perf_counter()
        dc = rs.deviceColumns(stream=0)
        t2 = time.perf_counter()
        res["device_exec_s"].append(t1 - t0)
        res["device_columns_s"].append(t2 - t1)
        return t2 - t0, rs, dc

    res = {"host_s": [], "device_s": [], "convert_ms": [], "kernel_ms": [], "rows_out": None, "parity": [], "device_exec_s": [],
           "device_columns_s": []}
    host_handoff()       # warm-up: module loads, pool growth, pinned-buffer cache
    device_handoff()
    res["device_exec_s"].clear()
    res["device_columns_s"].clear()
    for _ in range(runs):
        hs, hrs, cr = host_handoff()
        ds, drs, dc = device_handoff()
        assert drs.stats()["result_d2h_bytes"] == 0
        res["host_s"].append(hs)
        res["device_s"].append(ds)
        res["convert_ms"].append(dc.convert_ms())
        res["kernel_ms"].append(drs.kernel_ms())
        dcols = dc.to_host()
        plan = drs.getQueryMemDesc()
        parity(dcols, cr, plan.query_desc_type == abi.GroupByBaselineHash)
        res["parity"].append("ok")
        res["rows_out"] = dc.size()
        res["bytes_read"], res["bytes_written"] = conversion_bytes(plan, dc.size(), dcols)
        res["result_buffer_bytes"] = int(plan.buffer_size)
        del hrs, cr, drs, dc, dcols
    del keep, table
    torch.cuda.empty_cache()

    def stat(xs, scale=1.0):
        return {"mean": float(np.mean(xs)) * scale, "spread": float(np.max(xs) - np.min(xs)) * scale}
    conv_s = np.array(res["convert_ms"]) / 1e3
    moved = res["bytes_read"] + res["bytes_written"]
    return {"config": cfg, "rows": rows, "sql": sql, "rows_out": res["rows_out"], "result_buffer_bytes": res["result_buffer_bytes"],
            "host_handoff_ms": stat(res["host_s"], 1e3), "device_handoff_ms": stat(res["device_s"], 1e3),
            "device_execute_ms": stat(res["device_exec_s"], 1e3), "device_columns_call_ms": stat(res["device_columns_s"], 1e3),
            "scan_kernel_ms": stat(res["kernel_ms"]), "convert_kernel_ms": stat(res["convert_ms"]),
            "convert_bytes_read": res["bytes_read"], "convert_bytes_written": res["bytes_written"],
            "convert_tbs": float(np.mean(moved / conv_s)) / 1e12,
            "convert_share_of_read_ceiling": float(np.mean(moved / conv_s)) / 1e12 / READ_CEILING_TBS,
            "parity": res["parity"]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=float, default=1e9)
    ap.add_argument("--configs", default="c2,c4,c4s")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results to this file")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("result_handoff_bench needs a CUDA device (there is no CPU fallback)")
    torch.cuda.set_device(0)
    name, power = card()
    out = {"card": name, "power_limit": power, "runs": args.runs, "read_ceiling_tbs": READ_CEILING_TBS, "configs": []}
    for cfg in args.configs.split(","):
        r = run_config(cfg, int(args.rows), args.runs, torch)
        print(json.dumps(r), flush=True)
        out["configs"].append(r)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"card": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()
