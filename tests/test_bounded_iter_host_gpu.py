"""GPU: tests/cpp/bounded_iter_tests.cpp — GpuDB / ApplicationDB iterators with ReadOptions::iterate_upper_bound, with
and without ReadOptions::snapshot, and SeekForPrev, on a follower while replicated updates keep arriving."""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu


def test_bounded_iterators_through_the_host_mirror():
    if os.environ.get("RSP_TEST_EMUL_LIB"):
        pytest.skip("the C++ binary links librsp_b200.so")
    from rocksplicator_b200 import build
    exe = build.build_bounded_iter_tests()
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(p.stdout[-4000:], p.stderr[-2000:])
    assert p.returncode == 0 and " 0 failures" in p.stdout, p.stdout[-3000:]
