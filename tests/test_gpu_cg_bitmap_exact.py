"""Column-group bitmaps and bitmap-selected scans against the plain row-set model of tests/test_cg_bitmap_model.py.

Every device answer is compared with the model, never with another device path:
1. Folds (cgbm::fold_kernel): sequences of set / and / or from groups of different block sizes, at row offsets of every residue
   mod 32, two batches sharing a seam word, bitmaps of n_rows % 32 = 0 / 1 / 31 created all true or all false. Each fold source
   comes from a count path named by the kernel that ran: obgpu_count_kernel, obgpu_count_pipe_kernel<true> / <false>, the pipe
   kernel over 2000-row blocks, skip-index-settled blocks, a scan without a filter, and a filter-only scan whose result
   overflowed max_selected_rows. After every step fetch() equals the model bit for bit.
2. popcnt / fetch windows of every start and end residue, empty and inside one word; a 10 M-row all-true bitmap, larger than one
   grid of popcnt_kernel.
3. Bitmap-selected scans (obgpu_bitmap_slice_kernel, then every projection path): selected rows, per-block offsets, row ids,
   values (sign extension, unsigned images), NULL words and has_null, string lengths and bytes, fetch_strings, fetch_datums, the
   five aggregates and GROUP BY, with no row, every row, one row per block and empty blocks between dense ones selected.
4. Open paths: CS restated at open, LZ4 / zstd stored blocks, macro blocks, a device image without a host view.
5. A bitmap-selected result folded into a second bitmap.
6. Refusals: OB_INVALID_ARGUMENT, the bitmap bytes unchanged, and the context still usable."""
import contextlib
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import oracle_binding as ora
from test_aggregate_exact import COUNT, MAX, MIN, SUM, SUM_PRODUCT, exact_group_by_model
from test_aggregate_exact import fold as agg_fold
from test_cg_bitmap_model import (KINDS, N, OBJ, PLANS, STRING_KINDS, SWEEP, SWEEP_ROWS, block_starts, cells, column, fold,
                                  fold_steps, group_table, selection, values, white)
from test_gpu_scan_stage_records import kernels_run

pytestmark = pytest.mark.gpu
TESTS = os.path.dirname(os.path.abspath(__file__))

BASE = 0x10_0000_0000          # string_base: projected string pointers are BASE + offset in the caller's image


@pytest.fixture(scope="module")
def ob():
    import oceanbase_b200
    return oceanbase_b200


@pytest.fixture(scope="module")
def ctx(ob):
    c = ob.ScanContext(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def default_paths(monkeypatch):
    monkeypatch.delenv("OBGPU_PIPE", raising=False)
    monkeypatch.delenv("OBGPU_SPARSE_SPLIT", raising=False)


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in kv}
    for k, v in kv.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


class Batches:
    """page batches of the groups, opened once per module: plain, opened with OBGPU_PIPE=1, or with aggregate rows attached"""

    def __init__(self, ob, ctx):
        self.ob, self.ctx, self.open = ob, ctx, {}

    def get(self, kind, rpb, how="plain"):
        key = (kind, rpb, how)
        if key not in self.open:
            with env(OBGPU_PIPE="1" if how == "pipe1" else None):
                b = self.ctx.open_batch(group_table(kind, rpb))
            if how == "skip":
                b.set_agg_rows(*self.ob.table_agg_rows([column(kind)], [0], rpb))
            self.open[key] = b
        return self.open[key]

    def close(self):
        for b in self.open.values():
            b.close()


@pytest.fixture(scope="module")
def bs(ob, ctx):
    b = Batches(ob, ctx)
    yield b
    b.close()


def has(names, kernel):
    return any(kernel in k for k in names)


def traced(fn):
    """names of the kernels fn() launched. A trace without any kernel is taken again (a session can miss the launches right
    after it starts); every call traced here is a scan, freed, or a fold, and a fold applied again gives the same bits."""
    for _ in range(5):
        out = []

        def run():
            time.sleep(0.01)
            out.append(fn())
        names = kernels_run(run)
        if out[0] is not None:
            out[0].free()
        if names:
            return sorted(names)
    return []


def bits_of(words, k):
    j = np.arange(k)
    return ((words[j // 64] >> (j % 64).astype(np.uint64)) & np.uint64(1)).astype(bool)


# ---- fold sources ----------------------------------------------------------------------------------------------------------
def count_scan(bs, kind, rpb, fname, path):
    """the filter-only scan a fold step folds, on the count path `path` (test_cg_bitmap_model.PLANS)"""
    batch = bs.get(kind, rpb, {"big": "pipe1", "skip": "skip"}.get(path, "plain"))
    flt = None if fname is None else white(kind, fname)
    with env(OBGPU_PIPE={"pipe0": "0", "big": "1"}.get(path)):
        return batch.scan(flt, [], max_selected_rows=1 if path == "capped" else 0)


def assert_count_path(names, path):
    if path == "pipe0":
        assert has(names, "obgpu_count_kernel") and not has(names, "obgpu_count_pipe_kernel"), names
    elif path == "rec":
        assert has(names, "obgpu_count_pipe_kernel<true>"), names
    elif path in ("plan", "big"):
        assert has(names, "obgpu_count_pipe_kernel<false>") and not has(names, "obgpu_count_pipe_kernel<true>"), names
    elif path == "skip":
        assert has(names, "skip_index_kernel"), names
    elif path == "all":
        assert names and not has(names, "count"), names
    else:
        assert has(names, "count"), names


def fold_source(ob, bs, kind, rpb, fname, path):
    res = count_scan(bs, kind, rpb, fname, path)
    if path == "skip":
        f, t = res.skip_info()
        assert f > 0 and t > 0, (f, t)
    return res


def apply_checked(ob, bm, res, off, op, model, sel, what):
    """fold res into bm and the model; fetch() and popcnt() must equal the model afterwards"""
    bm.apply(res, off, op)
    fold(model, sel, off, op)
    got = bm.fetch().astype(bool)
    assert np.array_equal(got, model), (what, np.nonzero(got != model)[0][:8])
    assert bm.popcnt() == int(model.sum()), what


# ---- which kernels ran ---------------------------------------------------------------------------------------------------
# The kernel names come from torch.profiler in a short child process that runs the same scans (same tables, knobs, bitmaps, caps
# and row-id flag: the kernel choice is a function of those). A profiler session can come back without the launches near its
# start, and with this file's sessions in the suite's own process a later file's single-session kernel check came back empty;
# tracing in a child leaves the suite's process without a profiler session of this file's.
def count_key(kind, rpb, fname, path):
    return f"count:{kind}:{rpb}:{fname}:{path}"


def kernel_census():
    """{case: kernel names} for every count path of the fold plans, a fold, every bitmap-selected projection group and every
    generic / sparse-split case (run in the child process)"""
    import oceanbase_b200 as ob
    for k in ("OBGPU_PIPE", "OBGPU_SPARSE_SPLIT"):
        os.environ.pop(k, None)
    ctx = ob.ScanContext(0)
    bs = Batches(ob, ctx)
    out = {}
    try:
        for kind, rpb, fname, path, _, _ in fold_steps():
            key = count_key(kind, rpb, fname, path)
            if key not in out:
                count_scan(bs, kind, rpb, fname, path).free()          # first launch of each kernel outside the trace
                out[key] = traced(lambda: count_scan(bs, kind, rpb, fname, path))
        res = count_scan(bs, "int_dict", 133, "ge", "rec")
        bm = ob.CGBitmap(ctx, N + 40)
        bm.apply(res, 5, "or")
        out["fold"] = traced(lambda: bm.apply(res, 5, "or"))
        res.free()
        bm.free()
        for kind in KINDS:
            for rpb in (133, 2000):
                batch = bs.get(kind, rpb)
                bm = range_bitmap(ob, ctx, shape_bits("gaps", rpb, seed=3), 7, seed=4)
                batch.scan_bitmap(bm, proj_cols(kind), row_offset=7, want_row_ids=True).free()
                out[f"project:{kind}:{rpb}"] = traced(lambda: batch.scan_bitmap(bm, proj_cols(kind), row_offset=7, want_row_ids=True))
                bm.free()
        for kind in SPLIT_KINDS:
            for how in SPLIT_HOWS:
                _, _, batch, _, off, bm, cap = split_case(ob, ctx, bs, kind, how)
                with env(**SPLIT_KNOBS[how]):
                    batch.scan_bitmap(bm, proj_cols(kind), row_offset=off, want_row_ids=True, max_selected_rows=cap).free()
                    out[f"split:{kind}:{how}"] = traced(lambda: batch.scan_bitmap(bm, proj_cols(kind), row_offset=off, want_row_ids=True,
                                                                                  max_selected_rows=cap))
                bm.free()
    finally:
        bs.close()
        ctx.close()
    return out


@pytest.fixture(scope="module")
def census():
    root = os.path.dirname(TESTS)
    env_ = {k: v for k, v in os.environ.items() if k not in ("OBGPU_PIPE", "OBGPU_SPARSE_SPLIT")}
    env_["PYTHONPATH"] = os.pathsep.join([root, TESTS] + ([env_["PYTHONPATH"]] if env_.get("PYTHONPATH") else []))
    code = "import json, test_gpu_cg_bitmap_exact as t; print('CENSUS ' + json.dumps(t.kernel_census()))"
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, env=env_, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("CENSUS ")][-1][len("CENSUS "):])
    assert all(out.values()), [k for k, v in out.items() if not v]      # every case traced some kernel
    return out


@pytest.mark.parametrize("plan", PLANS + [("sweep", SWEEP_ROWS, False, SWEEP)], ids=lambda p: p[0])
def test_fold_sequences(ob, ctx, bs, census, plan):
    name, n_rows, all_true, steps = plan
    assert has(census["fold"], "fold_kernel"), census["fold"]
    bm = ob.CGBitmap(ctx, n_rows, all_true=all_true)
    model = np.full(n_rows, all_true)
    assert np.array_equal(bm.fetch().astype(bool), model) and bm.popcnt() == int(model.sum())
    sources = {}
    for kind, rpb, fname, path, off, op in steps:
        key = (kind, rpb, fname, path)
        assert_count_path(census[count_key(*key)], path)
        if key not in sources:
            sources[key] = fold_source(ob, bs, kind, rpb, fname, path)
        res = sources[key]
        what = (name, kind, rpb, fname, path, off, op)
        if path == "capped":
            # the result overflowed its capacity: its words must not be folded partially -- exact, or refused untouched
            before = bm.fetch()
            try:
                bm.apply(res, off, op)
            except ob.ObGpuError:
                assert np.array_equal(bm.fetch(), before), what
                continue
            fold(model, selection(kind, rpb, fname), off, op)
            assert np.array_equal(bm.fetch().astype(bool), model), what
            continue
        apply_checked(ob, bm, res, off, op, model, selection(kind, rpb, fname), what)
    for r in sources.values():
        r.free()
    bm.free()


# ---- popcnt / fetch --------------------------------------------------------------------------------------------------------
def pattern_bitmap(ob, ctx, bits, rpb=997):
    """a bitmap holding `bits`, written by folding (set) an EQ 1 scan of a 0/1 column whose rows are the bits"""
    t = ob.encode_table([ob.Column(ob.OBJ_INT, ob.ENC_RAW, bits.astype(np.int64))], rpb)
    b = ctx.open_batch(t)
    r = b.scan(ob.White(0, ob.WHITE_OP_EQ, (1,)), [])
    bm = ob.CGBitmap(ctx, len(bits))
    bm.apply(r, 0, "set")
    r.free()
    b.close()
    assert np.array_equal(bm.fetch().astype(bool), bits)
    return bm


def test_create_every_tail_residue(ob, ctx):
    for n in (0, 1, 2, 31, 32, 33, 63, 64, 65, 95, 1000, 1025):
        for all_true in (False, True):
            bm = ob.CGBitmap(ctx, n, all_true=all_true)
            assert bm.popcnt() == (n if all_true else 0)
            assert np.array_equal(bm.fetch()[:n], np.full(n, 1 if all_true else 0, dtype=np.uint8))
            if n:
                assert bm.popcnt(n - 1, n) == int(all_true)
            bm.free()


def test_popcnt_and_fetch_windows(ob, ctx):
    rng = np.random.default_rng(8)
    n = 161
    bits = rng.random(n) < 0.5
    bits[64:96] = True              # a full word, and a zero word next to it
    bits[96:128] = False
    bm = pattern_bitmap(ob, ctx, bits)
    pre = np.concatenate([[0], np.cumsum(bits)])
    for lo in range(0, 70):
        for hi in range(lo, min(lo + 70, n) + 1):
            assert bm.popcnt(lo, hi) == pre[hi] - pre[lo], (lo, hi)
    for lo in range(0, 98, 1):
        for cnt in (0, 1, 5, 31, 32, 33, 63, n - lo):
            if lo + cnt <= n:
                assert np.array_equal(bm.fetch(lo, cnt)[:cnt].astype(bool), bits[lo:lo + cnt]), (lo, cnt)
    bm.free()


def test_popcnt_beyond_one_grid(ob, ctx, bs):
    # 312 501 words: more than popcnt_kernel's 1024 x 256 threads, so its grid-stride loop runs
    n = 10_000_037
    bm = ob.CGBitmap(ctx, n, all_true=True)
    assert bm.popcnt() == n
    for lo, hi in ((n - 1, n), (n - 5, n), (n - 37, n), (n - 38, n - 1), (n - 64, n - 33), (1, n - 1), (33, n), (0, n - 5)):
        assert bm.popcnt(lo, hi) == hi - lo, (lo, hi)
    assert np.array_equal(bm.fetch(n - 100), np.ones(100, dtype=np.uint8))
    # a fold at the end of the range: its ragged last word is the bitmap's last word
    res = fold_source(ob, bs, "int_dict", 133, "ge", "rec")
    sel = selection("int_dict", 133, "ge")
    bm.apply(res, n - N, "and")
    assert bm.popcnt() == n - N + int(sel.sum())
    assert bm.popcnt(n - N, n) == int(sel.sum())
    assert np.array_equal(bm.fetch(n - N - 40).astype(bool), np.concatenate([np.ones(40, dtype=bool), sel]))
    for k in (1, 5, 31, 32, 33, 100):
        assert bm.popcnt(n - k, n) == int(sel[N - k:].sum()), k
    res.free()
    bm.free()


# ---- bitmap-selected scans -------------------------------------------------------------------------------------------------
def shape_bits(shape, rpb, seed):
    rng = np.random.default_rng(seed)
    st = block_starts(rpb)
    s = np.zeros(N, dtype=bool)
    if shape == "all":
        s[:] = True
    elif shape == "one_per_block":
        for b in range(len(st) - 1):
            s[st[b] + (7 * b) % (st[b + 1] - st[b])] = True
    elif shape == "gaps":            # dense blocks with empty ones between them
        s = rng.random(N) < 0.6
        for b in range(1, len(st) - 1, 3):
            s[st[b]:st[b + 1]] = False
    elif shape == "sparse":
        s = rng.random(N) < 0.03
    return s


def range_bitmap(ob, ctx, sel, off, seed, tail=9):
    """a bitmap of off + N + tail rows: sel at off, random bits around it (tail 0: the group's last row is the bitmap's)"""
    rng = np.random.default_rng(seed)
    bits = rng.random(off + N + tail) < 0.5
    bits[off:off + N] = sel
    return pattern_bitmap(ob, ctx, bits)


def check_projection(ob, res, kind, rpb, sel, image=None, string_base=BASE, aggregates=True):
    """a bitmap-selected result of group (kind, rpb) projecting [0] (and [0, 0] for integers), rows ids wanted, against the
    oracle's cells at the set bits of sel. image: the caller's image the string pointers address (None: not checked)"""
    c = cells(kind, rpb)
    rows = np.nonzero(sel)[0]
    k = len(rows)
    assert res.selected_rows == k, (kind, rpb)
    st = block_starts(rpb)
    so = res.fetch_sel_offsets()
    assert so[0] == 0 and np.array_equal(np.diff(so), [int(sel[st[b]:st[b + 1]].sum()) for b in range(len(st) - 1)])
    want = [c[i] for i in rows]
    null_want = np.array([x is None for x in want], dtype=bool)
    if k:
        rid = res.fetch_row_ids()
        blk = np.searchsorted(st, rows, side="right") - 1
        assert np.array_equal(st[blk] + rid, rows)
        data, lens, nulls = res.fetch_col(0)
        isnull = bits_of(nulls, k)
        assert np.array_equal(isnull, null_want), (kind, rpb)
        live = ~isnull
        if kind in STRING_KINDS:
            assert np.array_equal(lens[live], [len(x) for x in want if x is not None])
            heap, off = res.fetch_strings(0)
            got = [bytes(heap[off[j]:off[j + 1]]) for j in range(k)]
            assert [g for g, z in zip(got, isnull) if not z] == [x for x in want if x is not None], (kind, rpb)
            if image is not None:
                p = data.astype(np.int64) - string_base
                assert all(bytes(image[int(a):int(a) + len(x)]) == x for a, x, z in zip(p, want, isnull) if not z), (kind, rpb)
        else:
            el = res.col(0).elem_len
            mask = (1 << (8 * el)) - 1
            img = np.array([0 if x is None else x & mask for x in want], dtype=np.uint64)
            assert np.array_equal(data.astype(np.uint64)[live], img[live]), (kind, rpb)
    assert res.col(0).has_null == int(null_want.any()), (kind, rpb)
    if aggregates and kind not in STRING_KINDS:
        for agg in (COUNT, SUM, MIN, MAX):
            assert res.aggregate(agg, 0) == agg_fold(agg, want), (kind, rpb, agg)
        assert res.aggregate(SUM_PRODUCT, 0, 1) == agg_fold(SUM_PRODUCT, want, want), (kind, rpb)


def proj_cols(kind):
    return [0] if kind in STRING_KINDS else [0, 0]


REC_KINDS = {"int_dict", "vc_dict"}                     # flat dictionary columns: the record-path projection
PLAN_KINDS = {"int_auto", "int_raw_null", "vc_raw"}     # RLE / CONST blocks, RAW columns: the plan-path projection
SHAPES = [("none", 0, 9), ("all", 13, 0), ("one_per_block", 31, 9), ("gaps", 0, 9), ("gaps", 7, 0)]    # (shape, offset, tail)


@pytest.mark.parametrize("rpb", [133, 2000])
@pytest.mark.parametrize("kind", list(KINDS))
def test_bitmap_selected_projection(ob, ctx, bs, census, kind, rpb):
    names = census[f"project:{kind}:{rpb}"]
    assert has(names, "obgpu_bitmap_slice_kernel") and not has(names, "count"), names
    if rpb == 2000:
        assert has(names, "obgpu_project_kernel<false>"), names
    elif kind in REC_KINDS:
        assert has(names, "obgpu_project_pipe_kernel<true>"), names
    elif kind in PLAN_KINDS:
        assert has(names, "obgpu_project_pipe_kernel<false>"), names
    else:
        assert has(names, "project"), names
    t = group_table(kind, rpb)
    batch = bs.get(kind, rpb)
    image = None if kind == "vc_hex" else t.image      # HEX strings are rebuilt on the device: no image offset exists
    for i, (shape, off, tail) in enumerate(SHAPES):
        sel = shape_bits(shape, rpb, seed=i)
        bm = range_bitmap(ob, ctx, sel, off, seed=100 + i, tail=tail)
        res = batch.scan_bitmap(bm, proj_cols(kind), row_offset=off, want_row_ids=True, string_base=BASE)
        check_projection(ob, res, kind, rpb, sel, image)
        res.free()
        bm.free()


SPLIT_KINDS = ["int_raw_null", "tiny_dict", "u64_raw", "date_raw", "vc_dict", "vc_hex", "cs_str_dict"]
SPLIT_HOWS = ["pipe0", "hint_2000", "hint_pipe0", "split_env"]
SPLIT_KNOBS = {"pipe0": dict(OBGPU_PIPE="0"), "hint_2000": {}, "hint_pipe0": dict(OBGPU_PIPE="0"),
               "split_env": dict(OBGPU_PIPE="0", OBGPU_SPARSE_SPLIT="1")}


def split_case(ob, ctx, bs, kind, how):
    """(rpb, table, batch, selection, row offset, bitmap, max_selected_rows) of a generic / sparse-split projection case"""
    rpb = 2000 if how == "hint_2000" else 133
    shape, off = {"pipe0": ("gaps", 5), "hint_2000": ("sparse", 1), "hint_pipe0": ("one_per_block", 30), "split_env": ("gaps", 3)}[how]
    sel = shape_bits(shape, rpb, seed=7)
    bm = range_bitmap(ob, ctx, sel, off, seed=8)
    return rpb, group_table(kind, rpb), bs.get(kind, rpb), sel, off, bm, int(sel.sum()) if how.startswith("hint") else 0


@pytest.mark.parametrize("kind", SPLIT_KINDS)
@pytest.mark.parametrize("how", SPLIT_HOWS)
def test_generic_and_sparse_projection(ob, ctx, bs, census, kind, how):
    # pipe0: obgpu_project_kernel<false> at the small-block shape; hint_*: max_selected_rows <= total / 16 sends sparse blocks to
    # obgpu_project_sparse_kernel; split_env: OBGPU_SPARSE_SPLIT=1 does so for a dense selection
    names = census[f"split:{kind}:{how}"]
    if how == "pipe0":
        assert has(names, "obgpu_project_kernel<false>") and not has(names, "obgpu_project_sparse_kernel"), names
    else:
        assert has(names, "obgpu_project_kernel<true>") and has(names, "obgpu_project_sparse_kernel"), names
    rpb, t, batch, sel, off, bm, cap = split_case(ob, ctx, bs, kind, how)
    image = None if kind == "vc_hex" else t.image
    k = int(sel.sum())
    assert how not in ("hint_2000", "hint_pipe0") or k * 16 <= N
    with env(**SPLIT_KNOBS[how]):
        res = batch.scan_bitmap(bm, proj_cols(kind), row_offset=off, want_row_ids=True, string_base=BASE, max_selected_rows=cap)
        check_projection(ob, res, kind, rpb, sel, image)
        res.free()
        if k:      # one row short of the selection: the result reports the overflow instead of a partial answer
            short = batch.scan_bitmap(bm, proj_cols(kind), row_offset=off, want_row_ids=True, max_selected_rows=k - 1)
            with pytest.raises(ob.ObGpuError) as e:
                short.selected_rows
            assert e.value.code == ob.OB_BUF_NOT_ENOUGH
            short.free()
    bm.free()


def test_datums_under_a_bitmap(ob, ctx, bs):
    for kind in ("int_raw_null", "vc_dict"):
        t = group_table(kind, 133)
        sel = shape_bits("gaps", 133, seed=3)
        bm = range_bitmap(ob, ctx, sel, 11, seed=4)
        res = bs.get(kind, 133).scan_bitmap(bm, [0], row_offset=11, string_base=BASE)
        want = [x for x, s in zip(cells(kind, 133), sel) if s]
        k = len(want)
        datums, slots = res.fetch_datums(0)
        isnull = np.array([x is None for x in want])
        assert np.array_equal((datums["pack"] & ob.DATUM_NULL_BIT) != 0, isnull)
        if kind == "vc_dict":
            assert slots is None
            assert np.array_equal(datums["pack"][~isnull], [len(x) for x in want if x is not None])
            assert [bytes(t.image[int(p) - BASE:int(p) - BASE + len(x)]) for p, x in zip(datums["ptr"], want) if x is not None] == \
                [x for x in want if x is not None]
        else:
            assert np.all(datums["pack"][~isnull] == 8)
            assert np.array_equal(datums["ptr"], slots.ctypes.data + 8 * np.arange(k, dtype=np.uint64))
            assert np.array_equal(slots[~isnull], np.array([x & ((1 << 64) - 1) for x in want if x is not None], dtype=np.uint64))
        res.free()
        bm.free()


@pytest.mark.parametrize("kind", ["int_dict", "vc_dict", "cs_int_dict", "cs_str_dict"])
def test_group_by_under_a_bitmap(ob, ctx, bs, kind):
    aggs = [(COUNT, -1)] if kind in STRING_KINDS else [(COUNT, -1), (COUNT, 0), (SUM, 0), (MIN, 0), (MAX, 0)]
    st = block_starts(133)
    blocks = [ora.Block(group_table(kind, 133).block(b)) for b in range(len(st) - 1)]
    c = cells(kind, 133)
    for shape, off in (("gaps", 9), ("one_per_block", 0), ("none", 1)):
        sel = shape_bits(shape, 133, seed=5)
        bm = range_bitmap(ob, ctx, sel, off, seed=6)
        res = bs.get(kind, 133).scan_bitmap(bm, [0], row_offset=off)
        goff, out = res.group_by(0, aggs)
        for b, blk in enumerate(blocks):
            rows = np.nonzero(sel[st[b]:st[b + 1]])[0].astype(np.int32)
            want = exact_group_by_model(blk, 0, rows, aggs, {0: c[st[b]:st[b + 1]]})
            assert np.array_equal(out[:, goff[b]:goff[b + 1]], want), (kind, shape, b)
        res.free()
        bm.free()


# ---- open paths ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("how", ["cs_restated", "rebuilt", "lz4", "zstd", "macro", "device_no_view"])
def test_open_paths(ob, ctx, how):
    import torch
    from oceanbase_b200 import capi
    from oceanbase_b200.sstable import build_macro_blocks, compress_table
    from test_cs_stream_exact import encode_with
    kind = {"cs_restated": "cs_int", "rebuilt": "vc_hex", "lz4": "vc_dict", "zstd": "int_raw_null", "macro": "int_dict",
            "device_no_view": "vc_raw"}[how]
    fname = {"cs_restated": "gt", "rebuilt": "ge", "lz4": "in", "zstd": "lt", "macro": "ge", "device_no_view": "ge"}[how]
    rpb, keep, image = 133, None, None
    if how == "cs_restated":
        t = encode_with(5, [column(kind)], rpb)            # DELTA_ZIGZAG_PFOR streams, restated as RAW at open
        batch = ctx.open_batch(t)
    elif how in ("lz4", "zstd"):
        comp = capi.COMPRESSOR_LZ4 if how == "lz4" else capi.COMPRESSOR_ZSTD_1_3_8
        batch = ob.PageBatch(ctx, compress_table(group_table(kind, rpb), comp), compressor=comp)
    elif how == "macro":
        t = ob.encode_table([column(kind)], rpb, rowkey_cnt=1)     # sorted values: a valid rowkey
        mi = build_macro_blocks(t, [OBJ["int"]], 1, macro_block_size=64 << 10)
        batch = ob.PageBatch.from_macro_blocks(ctx, mi.image, 64 << 10, mi.n_macro)
    elif how == "device_no_view":
        t = group_table(kind, rpb)
        keep = torch.from_numpy(t.image).cuda()
        batch = ob.PageBatch(ctx, t, device_image_ptr=keep.data_ptr(), image_size=t.image.size, host_view=False)
        image = t.image                                 # string pointers address the caller's image, here on the device
    else:
        batch = ctx.open_batch(group_table(kind, rpb))      # HEX strings rebuilt at open: read back by fetch_strings only
    try:
        assert batch.n_blocks == len(block_starts(rpb)) - 1 and batch.total_rows == N
        # fold this batch's filter at an odd offset into a bitmap whose rows before it are set
        sel = selection(kind, rpb, fname)
        bm = ob.CGBitmap(ctx, N + 40, all_true=True)
        model = np.ones(N + 40, dtype=bool)
        res = batch.scan(white(kind, fname), [])
        apply_checked(ob, bm, res, 21, "and", model, sel, how)
        res.free()
        # and project it under that bitmap
        psel = model[21:21 + N]
        res = batch.scan_bitmap(bm, proj_cols(kind), row_offset=21, want_row_ids=True, string_base=BASE)
        check_projection(ob, res, kind, rpb, psel, image)
        res.free()
        bm.free()
    finally:
        batch.close()


# ---- chaining --------------------------------------------------------------------------------------------------------------
def test_bitmap_selected_result_folds_into_a_second_bitmap(ob, ctx, bs):
    res = fold_source(ob, bs, "int_dict", 500, "bt", "rec")
    bm1 = ob.CGBitmap(ctx, 2 * N + 9)
    m1 = np.zeros(2 * N + 9, dtype=bool)
    apply_checked(ob, bm1, res, N + 9, "set", m1, selection("int_dict", 500, "bt"), "first")
    res.free()
    # the second half of a two-range bitmap selects rows of another group; that result is folded into a second bitmap
    r2 = bs.get("vc_dict", 31).scan_bitmap(bm1, [0], row_offset=N + 9, want_row_ids=True)
    check_projection(ob, r2, "vc_dict", 31, m1[N + 9:], aggregates=False)
    bm2 = ob.CGBitmap(ctx, N + 33, all_true=True)
    m2 = np.ones(N + 33, dtype=bool)
    apply_checked(ob, bm2, r2, 19, "and", m2, m1[N + 9:], "chained and")
    r3 = fold_source(ob, bs, "tiny_dict", 133, "lt", "rec")
    apply_checked(ob, bm2, r3, 3, "or", m2, selection("tiny_dict", 133, "lt"), "chained or")
    r4 = bs.get("u64_raw", 2000).scan_bitmap(bm2, [0, 0], row_offset=33, want_row_ids=True)
    check_projection(ob, r4, "u64_raw", 2000, m2[33:33 + N])
    for r in (r2, r3, r4):
        r.free()
    bm1.free()
    bm2.free()


# ---- refusals --------------------------------------------------------------------------------------------------------------
def still_usable(ob, ctx, bs, bm, model):
    res = fold_source(ob, bs, "int_dict", 133, "ge", "rec")
    apply_checked(ob, bm, res, 0, "or", model, selection("int_dict", 133, "ge"), "after a refusal")
    res.free()
    r = bs.get("int_raw_null", 33).scan_bitmap(bm, [0, 0], row_offset=0, want_row_ids=True)
    check_projection(ob, r, "int_raw_null", 33, model[:N])
    r.free()


def test_refusals_leave_the_bitmap_and_context_intact(ob, ctx, bs):
    from oceanbase_b200 import capi
    lib = capi.lib
    n = N + 50
    bm = pattern_bitmap(ob, ctx, np.random.default_rng(9).random(n) < 0.5)
    model = bm.fetch().astype(bool)
    res = fold_source(ob, bs, "int_dict", 133, "ge", "rec")
    batch = bs.get("int_raw_null", 133)

    def refused(rc, what):
        assert rc == ob.OB_INVALID_ARGUMENT, (what, rc)
        assert np.array_equal(bm.fetch().astype(bool), model), what

    for op in (3, -1, 7):
        refused(lib.obgpu_cg_bitmap_apply_result(bm._h, res._h, 0, op), ("op", op))
    for off in (-1, n - N + 1, n, 1 << 62):
        refused(lib.obgpu_cg_bitmap_apply_result(bm._h, res._h, off, 1), ("apply offset", off))
        with pytest.raises(ob.ObGpuError) as e:
            batch.scan_bitmap(bm, [0], row_offset=off)
        assert e.value.code == ob.OB_INVALID_ARGUMENT
    cnt = C.c_int64(0)
    out = np.zeros(n + 8, dtype=np.uint8)
    for lo, hi in ((0, n + 1), (-1, 5), (6, 5), (n, n + 1)):
        refused(lib.obgpu_cg_bitmap_popcnt(bm._h, lo, hi, C.byref(cnt)), ("popcnt", lo, hi))
    for lo, k in ((n - 3, 4), (-1, 2), (0, n + 1), (3, -1)):
        refused(lib.obgpu_cg_bitmap_fetch(bm._h, lo, k, out.ctypes.data), ("fetch", lo, k))
    # a filter together with a bitmap: the bitmap is the selection, so the scan is refused
    f, keep = ob.flatten_filter(ob.White(0, ob.WHITE_OP_LT, (0,)))
    proj = (C.c_int32 * 1)(0)
    spec = capi.ScanSpec()
    spec.filter = C.pointer(f)
    spec.proj_cols, spec.n_proj = proj, 1
    h = C.c_void_p()
    refused(lib.obgpu_scan_bitmap(batch._h, bm._h, 0, C.byref(spec), C.byref(h)), "filter and bitmap")
    assert not h.value
    # a bitmap and a batch or result on different contexts
    ctx2 = ob.ScanContext(0)
    try:
        bm2 = ob.CGBitmap(ctx2, n, all_true=True)
        other = ctx2.open_batch(group_table("int_raw_null", 133))
        r_other = other.scan(white("int_raw_null", "lt"), [])
        refused(lib.obgpu_cg_bitmap_apply_result(bm._h, r_other._h, 0, 1), "result of another context")
        with pytest.raises(ob.ObGpuError) as e:
            other.scan_bitmap(bm, [0])
        assert e.value.code == ob.OB_INVALID_ARGUMENT
        assert lib.obgpu_cg_bitmap_apply_result(bm2._h, res._h, 0, 1) == ob.OB_INVALID_ARGUMENT
        with pytest.raises(ob.ObGpuError) as e:
            batch.scan_bitmap(bm2, [0])
        assert e.value.code == ob.OB_INVALID_ARGUMENT
        assert bm2.popcnt() == n
        r_other.free()
        other.close()
        bm2.free()
    finally:
        ctx2.close()
    # an empty range; a negative one is refused
    empty = ob.CGBitmap(ctx, 0, all_true=True)
    assert empty.popcnt() == 0 and empty.popcnt(0, 0) == 0 and len(empty.fetch(0, 0)) == 0
    assert lib.obgpu_cg_bitmap_popcnt(empty._h, 0, 1, C.byref(cnt)) == ob.OB_INVALID_ARGUMENT
    empty.free()
    h = C.c_void_p()
    assert lib.obgpu_cg_bitmap_create(ctx._h, -1, 0, C.byref(h)) == ob.OB_INVALID_ARGUMENT
    res.free()
    still_usable(ob, ctx, bs, bm, model)
    bm.free()


def test_model_inputs_are_the_written_values():
    # the model's cells are the generated values (tests/test_cg_bitmap_model.py checks every group; one here keeps the
    # device file honest when run alone)
    assert cells("u64_raw", 2000) == values("u64_raw")
