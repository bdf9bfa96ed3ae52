"""Integer stream codecs in CS column groups of the C++ compaction adapter (ObGpuColumnGroup::cs_stream_mode_ in
ObGpuPartitionMajorMerger::write_column_groups): tests/cpp/test_partition_merger_cs_streams.cpp writes the groups at stream mode 0,
plain and LZ4, and compares them with the host writer at mode 0; without a device it must refuse (exit 77)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "test_partition_merger_cs_streams")


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
def test_cs_stream_groups_equal_the_host_writer():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "partition merger cs stream tests passed" in r.stdout
