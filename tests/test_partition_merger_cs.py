"""CS column groups of the C++ compaction adapter (ObGpuColumnGroup::row_store_type_ = OB_GPU_CS_ENCODING_ROW_STORE in
ObGpuPartitionMajorMerger::write_column_groups): tests/cpp/test_partition_merger_cs.cpp checks a rowkey group and pure column
groups written as CS blocks, plain and compressed, against the host writer's CS encoding of the merged rows; without a device it
must refuse (exit 77)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "test_partition_merger_cs")


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
def test_cs_column_groups_equal_the_host_writer():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "partition merger cs tests passed" in r.stdout
