"""Device-resident results on a box without a GPU: the Arrow C Device Data Interface mirrors have the C compiler's layout,
`result_on_device` changes nothing in planning, and asking for device columns without a device is an error, not a
fallback to host code."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import ref_tables as rt
import sqlmini
from heavydb_b200 import abi, build, executor
from test_oracle_golden import COUNT_DISTINCT_QUERIES, FLOAT_QUERIES, MULTI_KEY_QUERIES, PATH_QUERIES, REFERENCE_QUERIES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_arrow_mirrors_match_c_compiler(tmp_path):
    build.build()
    fields = {
        "ArrowSchema": (abi.ArrowSchema, ["format", "name", "metadata", "flags", "n_children", "children", "dictionary", "release",
                                          "private_data"]),
        "ArrowArray": (abi.ArrowArray, ["length", "null_count", "offset", "n_buffers", "n_children", "buffers", "children",
                                        "dictionary", "release", "private_data"]),
        "ArrowDeviceArray": (abi.ArrowDeviceArray, ["array", "device_id", "device_type", "sync_event", "reserved"]),
        "B2QExecutionOptions": (abi.ExecutionOptions, ["device_ordinal", "result_on_device"]),
    }
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "b2q.h"\n#include "b2q_arrow.h"\nint main(){\n'
    for n, (_, fs) in fields.items():
        tag = n if n.startswith("B2Q") else f"struct {n}"
        prog += f'printf("{n} %zu\\n", sizeof({tag}));\n'
        for f in fs:
            prog += f'printf("{n}.{f} %zu\\n", offsetof({tag}, {f}));\n'
    prog += 'printf("ARROW_DEVICE_CUDA %d\\n", ARROW_DEVICE_CUDA);\nprintf("ARROW_FLAG_NULLABLE %d\\n", ARROW_FLAG_NULLABLE);\n'
    prog += 'printf("STAT %d\\n", B2Q_STAT_RESULT_D2H_BYTES);\nprintf("ABI %d\\n", B2Q_ABI_VERSION);\nreturn 0;}\n'
    src = tmp_path / "arrow_sz.c"
    src.write_text(prog)
    exe = tmp_path / "arrow_sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)]).decode().splitlines())
    for n, (cls, fs) in fields.items():
        assert int(out[n]) == C.sizeof(cls), n
        for f in fs:
            assert int(out[f"{n}.{f}"]) == getattr(cls, f).offset, f"{n}.{f}"
    assert int(out["ARROW_DEVICE_CUDA"]) == abi.ARROW_DEVICE_CUDA
    assert int(out["ARROW_FLAG_NULLABLE"]) == abi.ARROW_FLAG_NULLABLE
    assert int(out["STAT"]) == abi.STAT_RESULT_D2H_BYTES
    assert int(out["ABI"]) == abi.ABI_VERSION == executor.lib().b2q_abi_version()


def test_plan_does_not_depend_on_result_on_device():
    table = rt.make_table(rt.test_rows())
    ex = executor.Executor()
    checked = 0
    def outcome(unit, hint, on):
        try:
            return bytes(ex.plan(unit, table, eo=executor.execution_options(output_columnar_hint=hint, result_on_device=on)))
        except executor.QueryExecutionError as e:   # a unit the planner refuses is refused either way
            return e.code

    for sql in REFERENCE_QUERIES + MULTI_KEY_QUERIES + PATH_QUERIES + COUNT_DISTINCT_QUERIES + FLOAT_QUERIES:
        unit = sqlmini.parse(sql, table, rt.TEST_NAMES)
        for hint in (False, True):
            off, on = outcome(unit, hint, False), outcome(unit, hint, True)
            assert off == on, sql
            checked += isinstance(off, bytes)
    assert checked >= 40


def test_result_on_device_flag_reaches_the_library():
    eo = executor.execution_options(result_on_device=True)
    assert eo.result_on_device == 1
    assert executor.execution_options().result_on_device == 0


def _no_device():
    if executor.lib().b2q_device_count() > 0:
        pytest.skip("a CUDA device is present")


def test_device_columns_without_a_device_is_an_error_not_a_fallback():
    """A host-resident result set (wrapped storage, no device involved) still cannot be converted on the host by this
    entry: it answers B2Q_ERR_NO_DEVICE, hands out no handle, and the host read-out keeps working."""
    _no_device()
    table = rt.make_table(rt.test_rows())
    unit = sqlmini.parse("SELECT x, COUNT(*), SUM(y) FROM test GROUP BY x;", table, rt.TEST_NAMES)
    ex = executor.Executor()
    plan = ex.plan(unit, table)
    rs = ex.resultSetFromStorage(np.zeros(plan.buffer_size, dtype=np.uint8), unit, table)
    h = C.c_void_p()
    rc = executor.lib().b2q_rs_device_columns(rs._h, None, C.byref(h))
    assert rc == abi.ERR_NO_DEVICE and not h.value
    with pytest.raises(executor.NoDeviceError):
        rs.deviceColumns(stream=0)
    assert rs.stats()["result_d2h_bytes"] == 0
    assert len(rs.columnarResults()) == 3
    with pytest.raises(executor.NoDeviceError):
        ex.executeWorkUnit(0, True, table, unit, result_on_device=True)
