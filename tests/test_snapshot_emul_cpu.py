"""CPU-only: tests/test_snapshot_gpu.py and tests/emul/fuzz_snapshots_vs_port.py against the CPU emulation build of the
engine (tests/emul/build_emul.py), in a subprocess, as tests/test_emul_cpu.py does for the parity suite.  This catches
logic and addressing bugs of the snapshot paths before GPU time is spent; the `-m gpu` run on an H100 is the real test."""
import importlib.util
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul():
    spec = importlib.util.spec_from_file_location("build_emul", os.path.join(ROOT, "tests", "emul", "build_emul.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build()


def test_snapshot_suite_under_emulation(emul):
    env = dict(os.environ)
    env["RSP_TEST_EMUL_LIB"] = emul[0]
    env.setdefault("RSP_TEST_EMUL_ARENA", str(16 << 20))
    p = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider",
                        "tests/test_snapshot_gpu.py"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-3000:]


def test_snapshots_vs_port_fuzz_under_emulation(emul):
    env = dict(os.environ)
    env["RSP_TEST_EMUL_LIB"] = emul[0]
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emul", "fuzz_snapshots_vs_port.py"), "0", "36"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    print(p.stdout[-2000:], p.stderr[-2000:])
    assert p.returncode == 0 and "done bad= 0" in p.stdout
