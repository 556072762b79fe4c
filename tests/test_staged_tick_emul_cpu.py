"""CPU-only: tests/test_staged_tick_gpu.py against the CPU emulation build of the engine (tests/emul/build_emul.py), in a
subprocess, as tests/test_emul_cpu.py does for the parity suite.  The `-m gpu` run on an H100 is the real test."""
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


def test_staged_tick_under_emulation(emul):
    env = dict(os.environ)
    env["RSP_TEST_EMUL_LIB"] = emul[0]
    env.setdefault("RSP_TEST_EMUL_ARENA", str(16 << 20))
    p = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider",
                        "tests/test_staged_tick_gpu.py"], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0 and "1 passed" in p.stdout, p.stdout[-3000:]
