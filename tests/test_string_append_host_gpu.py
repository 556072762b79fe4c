"""GPU: tests/cpp/string_append_tests.cpp — rocksdb::StringAppendOperator (delimiters ',', '\\0' and none) through
GpuDB::Open, which maps it to the device operator, and ApplicationDB: Write(Merge), Get, MultiGet, iterators, reads at
snapshots, Backup / Restore with the folded values in the SST."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def test_string_append_through_the_host_mirror():
    if os.environ.get("RSP_TEST_EMUL_LIB"):
        pytest.skip("the C++ binary links librsp_b200.so")
    from rocksplicator_b200 import build
    exe = build.build_string_append_tests()
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(p.stdout[-4000:], p.stderr[-2000:])
    assert p.returncode == 0 and " 0 failures" in p.stdout, p.stdout[-3000:]
