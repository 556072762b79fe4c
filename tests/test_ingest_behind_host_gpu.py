"""GPU: tests/cpp/ingest_behind_tests.cpp — Options::allow_ingest_behind, IngestExternalFileOptions::ingest_behind and
CompactRange(change_level) through GpuDB::Open and ApplicationDB, step for step as the reference's
application_db_test.cpp:300-342, then a backfill below existing writes."""
import os
import subprocess
import tempfile

import pytest

pytestmark = pytest.mark.gpu


def test_ingest_behind_through_the_host_mirror():
    if os.environ.get("RSP_TEST_EMUL_LIB"):
        pytest.skip("the C++ binary links librsp_b200.so")
    from rocksplicator_b200 import build
    exe = build.build_ingest_behind_tests()
    with tempfile.TemporaryDirectory() as d:
        p = subprocess.run([exe, d], capture_output=True, text=True, timeout=600)
    print(p.stdout[-4000:], p.stderr[-2000:])
    assert p.returncode == 0 and " 0 failures" in p.stdout, p.stdout[-3000:]
