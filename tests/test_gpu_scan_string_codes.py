"""Batch string codes (batch_codes.cuh): an EQ / NE / IN leaf on a dictionary-coded VARCHAR / CHAR column scanned with stage records
is evaluated once per scan over the batch's distinct strings, and the count kernel looks each row's code up in that bitset. Every
scan here runs with the codes on and with them off (OBGPU_STR_CODES=0: the per-block dictionary leaf) and is checked against the
plain bytes model of tests/test_string_filter_exact.py: selection and every projected column.

Covered: every EQ / NE / IN leaf of the model's edge constants (absent constants, the empty string, strings sharing their length and
first 8 bytes), NULL rows, OR trees and AND trees whose string leaf is not the first, several batches scanned more than once and a
batch closed and opened again, and a column above the 65 536-code cap (it keeps the per-block path)."""
import ctypes as C

import numpy as np
import pytest

from test_string_filter_exact import EQ, IN, NE, OBJ_INT, OBJ_VARCHAR, S, leaves, selected, spec_of, table_of, trees
from test_gpu_string_filter_exact import PROJ, check_scan

pytestmark = pytest.mark.gpu

EQ_OPS = (EQ, NE, IN)


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


def codes_state(ob, batch, col=S):
    state, n, ms = C.c_int32(), C.c_int32(), C.c_float()
    assert ob.capi.lib.obgpu_batch_string_codes(batch._h, col, C.byref(state), C.byref(n), C.byref(ms)) == 0
    return state.value, n.value


def eq_cases(spec):
    """every string equality leaf and every tree of the model (trees mix the string leaf with an integer leaf, AND and OR)"""
    out = [(n, f) for n, f in leaves(spec) if getattr(f, "op", None) in EQ_OPS and getattr(f, "col", None) == S]
    return out + trees(spec)


def check_both(ob, batch, spec, monkeypatch, cases):
    wants = [selected(spec, f) for _, f in cases]
    for knob in ("1", "0"):
        monkeypatch.setenv("OBGPU_STR_CODES", knob)
        for j, ((name, f), want) in enumerate(zip(cases, wants)):
            check_scan(batch, spec, (knob, name), f, True, want)


@pytest.fixture(autouse=True)
def pipe(monkeypatch):
    monkeypatch.setenv("OBGPU_PIPE", "1")


@pytest.mark.parametrize("tname,nname", [("varchar", "n0"), ("varchar", "n10"), ("char", "n10"), ("varchar", "n100")])
def test_codes_match_the_bytes_model(ob, ctx, monkeypatch, tname, nname):
    spec = spec_of("dict_var", tname, nname)
    batch = ctx.open_batch(table_of("dict_var", tname, nname))
    try:
        check_both(ob, batch, spec, monkeypatch, eq_cases(spec))
        state, n = codes_state(ob, batch)
        assert state == 1 and n >= 1 if nname != "n100" else state in (0, 1), (state, n)
    finally:
        batch.close()


def test_several_batches_rescanned_and_reopened(ob, ctx, monkeypatch):
    specs = [spec_of("dict_var", "varchar", "n10"), spec_of("dict_var", "char", "n0")]
    tables = [table_of("dict_var", "varchar", "n10"), table_of("dict_var", "char", "n0")]
    for _ in range(2):   # open, scan twice, close; then again
        batches = [ctx.open_batch(t) for t in tables]
        try:
            for _ in range(2):
                for spec, batch in zip(specs, batches):
                    cases = eq_cases(spec)[::3]
                    monkeypatch.setenv("OBGPU_STR_CODES", "1")
                    for name, f in cases:
                        check_scan(batch, spec, name, f, True)
            for batch in batches:
                assert codes_state(ob, batch)[0] == 1
        finally:
            for batch in batches:
                batch.close()


def test_column_over_the_code_cap_keeps_the_region_path(ob, ctx, monkeypatch):
    n = 70_000
    vals = [b"v%07d" % i + b"x" * (i % 3) for i in range(n)]   # variable lengths: a dict_var dictionary in every block
    cols = [ob.Column(OBJ_INT, 0, np.arange(n, dtype=np.int64)), ob.Column(OBJ_VARCHAR, 1, vals)]   # RAW, DICT: all distinct
    batch = ctx.open_batch(ob.encode_table(cols, 133))
    try:
        monkeypatch.setenv("OBGPU_STR_CODES", "1")
        for f, want in ((ob.White(1, EQ, (b"v0069999",)), [69_999]), (ob.White(1, IN, (b"v0000003", b"nope")), [3]),
                        (ob.White(1, NE, (b"v0000000",)), list(range(1, n)))):
            res = batch.scan(f, [0])
            assert res.selected_rows == len(want)
            assert [int(x) for x in res.fetch_col(0)[0]] == want
            res.free()
        assert codes_state(ob, batch, 1)[0] == -2   # OBGPU_CODES_OVER_CAP
    finally:
        batch.close()
