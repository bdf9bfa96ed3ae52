"""The table tests/test_gpu_pipeline_group_by.py groups through the host pipeline to show that the 65 536-value cap of
obgpu_result_group_by_values applies per page batch, built here on the CPU, and proof from the block bytes (the dictionaries read
through the oracle) that its dictionaries hold more than 65 536 distinct values in all while every batch of CAP_SPLIT blocks holds
fewer."""
import functools

import numpy as np

from test_group_by_columns_shapes import dict_values
from test_scan_codes_model import CAP

CAP_ROWS, CAP_RPB = 160_000, 2000
CAP_SPLIT = 40          # blocks per batch: 40 000 distinct values each


@functools.lru_cache(maxsize=None)
def cap_split_table():
    """0 row id (RAW); 1 INT DICT row id // 2: 80 000 distinct values, 1 000 per block"""
    import oceanbase_b200 as ob
    i = np.arange(CAP_ROWS, dtype=np.int64)
    return ob.encode_table([ob.Column(ob.OBJ_INT, ob.ENC_RAW, i), ob.Column(ob.OBJ_INT, ob.ENC_DICT, i // 2)], CAP_RPB)


@functools.lru_cache(maxsize=None)
def cap_split_cells():
    i = list(range(CAP_ROWS))
    return [i, [r // 2 for r in i]]


def test_cap_split_table_is_over_the_cap_in_all_and_under_it_per_batch():
    t = cap_split_table()
    assert t.n_blocks == CAP_ROWS // CAP_RPB and t.n_blocks % CAP_SPLIT == 0
    per_batch = [dict_values(t, 1, range(b, b + CAP_SPLIT)) for b in range(0, t.n_blocks, CAP_SPLIT)]
    assert all(len(v) <= CAP for v in per_batch) and len(per_batch) >= 2
    assert len(set().union(*per_batch)) > CAP
    cells = cap_split_cells()
    assert len(set(cells[1])) == len(set().union(*per_batch))


# ---- a different shared-memory fold per page batch ----------------------------------------------------------------------------
RANK_BYTES = 8 * 256 * 4          # group_values.cuh kRankBytes: a CTA's rank arrays of one group column
SHARED_ACC_BUDGET = 48 << 10
VARY_RPB, VARY_BLOCKS = 100, 48
VARY_AGGS = 3                     # the GPU test's COUNT(*), SUM, MAX


def vary_dicts(b):
    """block b's distinct values of group columns 1 and 2"""
    return 2 + (b * 7) % 40, 2 + (b * 3) % 8


@functools.lru_cache(maxsize=None)
def vary_table():
    """0 row id (RAW); 1 INT DICT r % d1(b); 2 INT DICT r % d2(b): every block has dictionaries of its own size"""
    import oceanbase_b200 as ob
    i = np.arange(VARY_RPB * VARY_BLOCKS, dtype=np.int64)
    d1 = np.repeat([vary_dicts(b)[0] for b in range(VARY_BLOCKS)], VARY_RPB)
    d2 = np.repeat([vary_dicts(b)[1] for b in range(VARY_BLOCKS)], VARY_RPB)
    return ob.encode_table([ob.Column(ob.OBJ_INT, ob.ENC_RAW, i), ob.Column(ob.OBJ_INT, ob.ENC_DICT, i % d1),
                            ob.Column(ob.OBJ_INT, ob.ENC_DICT, i % d2)], VARY_RPB)


@functools.lru_cache(maxsize=None)
def vary_cells():
    i = list(range(VARY_RPB * VARY_BLOCKS))
    return [i, [r % vary_dicts(r // VARY_RPB)[0] for r in i], [r % vary_dicts(r // VARY_RPB)[1] for r in i]]


def test_vary_table_takes_the_shared_fold_with_a_different_size_per_batch():
    t = vary_table()
    assert t.n_blocks == VARY_BLOCKS
    for bpb in (1, 2):
        smem = set()
        for b in range(0, VARY_BLOCKS, bpb):
            blocks = range(b, min(b + bpb, VARY_BLOCKS))
            p = (len(dict_values(t, 1, blocks)) + 1) * (len(dict_values(t, 2, blocks)) + 1)
            acc = p * (VARY_AGGS + 1) * 16
            assert acc <= SHARED_ACC_BUDGET                  # the shared path: its dynamic shared memory depends on P
            smem.add(2 * RANK_BYTES + acc)
        assert len(smem) >= 10, bpb
