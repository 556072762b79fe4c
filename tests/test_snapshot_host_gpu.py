"""GPU: tests/cpp/snapshot_tests.cpp — GpuDB / ApplicationDB reads with ReadOptions::snapshot stay as they were while
later updates arrive through RocksDBReplicator; IngestExternalFile with snapshot_consistency = false while a snapshot is
live answers NotSupported."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def test_snapshot_reads_through_the_host_mirror():
    if os.environ.get("RSP_TEST_EMUL_LIB"):
        pytest.skip("the C++ binary links librsp_b200.so")
    from rocksplicator_b200 import build
    exe = build.build_snapshot_tests()
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(p.stdout[-4000:], p.stderr[-2000:])
    assert p.returncode == 0 and " 0 failures" in p.stdout, p.stdout[-3000:]
