"""The per-column encodings of the C++ compaction adapter (ObGpuColumnGroup::encodings_ in
ObGpuPartitionMajorMerger::write_column_groups): tests/cpp/test_partition_merger_encodings.cpp checks every column group written
with OBGPU_ENC_AUTO, host-spliced blocks included, plain and compressed, against the host writer's AUTO encoding of the merged
rows; without a device it must refuse (exit 77)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "test_partition_merger_encodings")


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
def test_auto_column_groups_equal_the_host_writer():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "partition merger encodings tests passed" in r.stdout
