"""Runtime interrupt and dynamic watchdog at the boundary, without a GPU: the new symbols are exported, the ctypes mirror of
B2QExecutionOptions has the C layout with the new fields, a token cannot be made without a device, the options do not change
a plan, and the error-precedence rule (Execute.cpp:2319-2324) holds."""
import ctypes as C
import os
import subprocess

import pytest

import oracle_lib
import ref_tables as rt
from heavydb_b200 import abi, build, executor, sqlmini

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = ["b2q_interrupt_token_create", "b2q_interrupt_token_destroy", "b2q_interrupt", "b2q_interrupt_reset", "b2q_interrupt_is_set"]


@pytest.fixture(scope="module")
def libpath():
    return build.build()


def test_symbols_exported(libpath):
    lib = C.CDLL(libpath)
    assert all(hasattr(lib, n) for n in SYMBOLS)
    assert lib.b2q_abi_version() == abi.ABI_VERSION == 9


def test_execution_options_layout(tmp_path):
    fields = ["result_on_device", "with_dynamic_watchdog", "dynamic_watchdog_time_limit", "allow_runtime_query_interrupt", "interrupt_token"]
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "b2q.h"\nint main(){\n'
    prog += 'printf("size %zu\\n", sizeof(B2QExecutionOptions));\n'
    for f in fields:
        prog += f'printf("{f} %zu\\n", offsetof(B2QExecutionOptions, {f}));\n'
    prog += "return 0;}\n"
    src = tmp_path / "eo.c"
    src.write_text(prog)
    exe = tmp_path / "eo"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    out = dict(line.split() for line in subprocess.check_output([str(exe)]).decode().splitlines())
    assert int(out["size"]) == C.sizeof(abi.ExecutionOptions)
    for f in fields:
        assert int(out[f]) == getattr(abi.ExecutionOptions, f).offset, f
    # appended: a zero-initialised caller keeps the old behaviour
    eo = abi.ExecutionOptions()
    assert (eo.with_dynamic_watchdog, eo.dynamic_watchdog_time_limit, eo.allow_runtime_query_interrupt, eo.interrupt_token) == (0, 0, 0, None)


@pytest.mark.skipif(executor.lib().b2q_device_count() > 0, reason="checks the CPU-only refusal")
def test_token_without_device_is_refused():
    h = C.c_void_p()
    assert executor.lib().b2q_interrupt_token_create(C.byref(h)) == abi.ERR_NO_DEVICE
    assert not h.value
    with pytest.raises(executor.NoDeviceError):
        executor.InterruptToken()
    # a NULL token is harmless everywhere
    L = executor.lib()
    L.b2q_interrupt(None)
    L.b2q_interrupt_reset(None)
    L.b2q_interrupt_token_destroy(None)
    assert L.b2q_interrupt_is_set(None) == 0


SQLS = ["SELECT COUNT(*), SUM(x) FROM test WHERE y > 41;", "SELECT x, COUNT(*), AVG(y) FROM test GROUP BY x;",
        "SELECT t, SUM(y), MIN(d) FROM test GROUP BY t;", "SELECT x, y FROM test WHERE z > 101 LIMIT 3"]


@pytest.mark.parametrize("sql", SQLS)
def test_options_do_not_change_plans(sql):
    table = rt.make_table(rt.test_rows())
    unit = sqlmini.parse(sql, table, rt.TEST_NAMES)
    ex = executor.Executor()
    off = ex.plan(unit, table, max_groups_buffer_entry_guess=48, has_cardinality_estimation=True).as_dict()
    eo = executor.execution_options(with_dynamic_watchdog=True, dynamic_watchdog_time_limit=1, allow_runtime_query_interrupt=True)
    on = ex.plan(unit, table, eo=eo, max_groups_buffer_entry_guess=48, has_cardinality_estimation=True).as_dict()
    assert on == off
    if unit.unit.num_target_exprs and "LIMIT" not in sql:
        assert oracle_lib.plan(unit, table, entry_guess=48, has_card=True).as_dict() == on


@pytest.mark.parametrize("code,watchdog,interrupted,want", [
    (abi.ERR_OUT_OF_TIME, True, True, abi.ERR_INTERRUPTED),      # Execute.cpp:2319-2324
    (abi.ERR_OUT_OF_TIME, True, False, abi.ERR_OUT_OF_TIME),
    (abi.ERR_OUT_OF_TIME, False, True, abi.ERR_OUT_OF_TIME),     # the rule needs the watchdog on
    (abi.ERR_INTERRUPTED, True, True, abi.ERR_INTERRUPTED),
    (abi.ERR_INTERRUPTED, False, False, abi.ERR_INTERRUPTED),
    (abi.ERR_OUT_OF_SLOTS, True, True, abi.ERR_OUT_OF_SLOTS),    # other errors keep their code
    (abi.OK, True, True, abi.OK),
])
def test_error_precedence(code, watchdog, interrupted, want):
    assert executor.resolve_interrupt_error(code, watchdog, interrupted) == want


@pytest.mark.parametrize("code", [abi.ERR_OUT_OF_TIME, abi.ERR_INTERRUPTED])
def test_codes_map_to_query_execution_error(code):
    with pytest.raises(executor.QueryExecutionError) as ei:
        executor._raise(code)
    assert ei.value.code == code
    assert type(ei.value) is executor.QueryExecutionError
    assert executor.lib().b2q_error_string(code).decode() in (
        "Query execution has exceeded the time limit", "Query execution has been interrupted")
