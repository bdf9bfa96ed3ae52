"""The skip-index columns of the C++ compaction adapter (ObGpuColumnGroup::skip_index_cols_):
tests/cpp/test_partition_merger_agg_rows.cpp checks that write_column_groups returns every block's aggregate row, host-spliced
blocks included, byte for byte what the host writer's obgpu_writer_table_agg_rows builds over the group's rows; without a
device it must refuse (exit 77)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "test_partition_merger_agg_rows")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_builds_and_refuses_without_device():
    assert os.path.exists(BIN)  # built by __graft_entry__.build()
    if _has_gpu():
        pytest.skip("device present: covered by the gpu test")
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=120)
    assert r.returncode == 77, r.stdout + r.stderr


@pytest.mark.gpu
def test_column_group_agg_rows_equal_the_host_writer():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "partition merger agg rows tests passed" in r.stdout
