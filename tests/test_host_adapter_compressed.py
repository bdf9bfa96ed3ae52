"""C++ host adapter over stored (compressed) micro-blocks: tests/cpp/test_host_adapter_compressed.cpp scans LZ4, zstd and zlib
tables through ObGpuSSTableBatchScanner::set_compressor (single batch and pipelined) and ObGpuStoreRowIterator and compares them
with the same scans of the plain image; without a device it must refuse (exit 77)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "test_host_adapter_compressed")


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_compressed_adapter_builds_and_refuses_without_device():
    assert os.path.exists(BIN)  # built by __graft_entry__.build()
    if _has_gpu():
        pytest.skip("device present: covered by the gpu test")
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=120)
    assert r.returncode == 77, r.stdout + r.stderr


@pytest.mark.gpu
def test_compressed_adapter_parity_on_gpu():
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert "compressed host adapter tests passed" in r.stdout
