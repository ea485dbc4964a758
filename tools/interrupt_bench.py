"""Cost and latency of the runtime interrupt and the dynamic watchdog on 1e9-row bench workloads (one GPU).

    python tools/interrupt_bench.py [--configs c2,c2all,c3,c4,c4s] [--reps 3] [--latency-runs 5] [--out FILE]

kernel_overhead: per config, the scan's CUDA-event time with the feature off and with it on but never triggered (an interrupt
token that is never set + a 10 s watchdog), the two alternating in one process, mean of --reps each.
interrupt_latency: c4 at 1e9 rows, a timer thread interrupts the call 10 ms after it starts; median of --latency-runs of the
time from b2q_interrupt to the call's return.  The card's name and power limit are read in the same run and printed with
the numbers.  Tables are generated in HBM by bench.py's generator (a ring of 4 resident 32 Mi-row fragments).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from heavydb_b200 import abi, executor  # noqa: E402


def card():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception as e:  # read-only query; report why it is missing
        info["power_limit_w"] = f"unknown ({e.__class__.__name__})"
    return info


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c2all,c3,c4,c4s")
    ap.add_argument("--rows", type=int, default=10**9)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--latency-runs", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    ex = executor.Executor()
    tok = executor.InterruptToken()
    off = executor.execution_options()
    on = executor.execution_options(allow_runtime_query_interrupt=True, interrupt_token=tok, with_dynamic_watchdog=True,
                                    dynamic_watchdog_time_limit=10_000)
    result = {"card": card(), "rows": args.rows, "kernel_overhead": {}, "interrupt_latency": {}}
    tables = {}
    for cfg in args.configs.split(","):
        frags = bench.rank_fragments(args.rows, 0, 1, ring=4)
        table, keep = bench.build_device_table(cfg, frags, torch)
        names = [c[0] for c in bench.CONFIGS[cfg][0]]
        unit = bench.make_unit(cfg, bench.CONFIGS[cfg][1], table, names)
        guess = bench.ENTRY_GUESS.get(cfg, 0)
        bt = table.build(abi.GPU_LEVEL)
        run = lambda eo: ex.executeWorkUnit(guess, True, bt, unit, eo=eo, has_cardinality_estimation=guess > 0,
                                            memory_level=abi.GPU_LEVEL)
        run(off), run(on)  # warm-up
        t_off, t_on = [], []
        for _ in range(args.reps):
            t_off.append(run(off).kernel_ms())
            t_on.append(run(on).kernel_ms())
        m_off, m_on = statistics.mean(t_off), statistics.mean(t_on)
        result["kernel_overhead"][cfg] = {"off_ms": round(m_off, 3), "on_ms": round(m_on, 3),
                                         "overhead_pct": round(100.0 * (m_on - m_off) / m_off, 2),
                                         "off_all": [round(x, 3) for x in t_off], "on_all": [round(x, 3) for x in t_on]}
        print(cfg, result["kernel_overhead"][cfg], flush=True)
        tables[cfg] = (bt, keep, unit, guess)
        if cfg != "c4":
            del keep
            tables.pop(cfg)
            torch.cuda.empty_cache()

    if "c4" in tables:
        bt, _keep, unit, guess = tables["c4"]
        lat = []
        for _ in range(args.latency_runs):
            tok.reset()
            fired = {}

            def fire():
                time.sleep(0.010)
                fired["t"] = time.perf_counter()
                tok.interrupt()

            th = threading.Thread(target=fire)
            th.start()
            code = 0
            try:
                ex.executeWorkUnit(guess, True, bt, unit, eo=on, memory_level=abi.GPU_LEVEL)
            except executor.QueryExecutionError as e:
                code = e.code
            t1 = time.perf_counter()
            th.join()
            lat.append({"code": code, "interrupt_to_return_ms": round((t1 - fired["t"]) * 1e3, 3)})
        tok.reset()
        ok = [x["interrupt_to_return_ms"] for x in lat if x["code"] == abi.ERR_INTERRUPTED]
        result["interrupt_latency"]["c4"] = {"runs": lat, "median_ms": statistics.median(ok) if ok else None}
        print("c4 latency", result["interrupt_latency"]["c4"], flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
