"""CPU-only: tests/test_lookup_collisions_gpu.py against the CPU emulation build of the engine (tests/emul/build_emul.py),
in a subprocess, as tests/test_streams_emul_cpu.py does for the stream suite.  The emulation runs the kernels' own
probe loops, so every collision scenario runs here; it serialises atomics, so the insert races of the same-tick
collisions (M5) are exercised by the `-m gpu` run on an H100 alone."""
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


def test_collision_suite_under_emulation(emul):
    env = dict(os.environ)
    env["RSP_TEST_EMUL_LIB"] = emul[0]
    env.setdefault("RSP_TEST_EMUL_ARENA", str(16 << 20))
    p = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-q", "-p", "no:cacheprovider", "-rs",
                        "tests/test_lookup_collisions_gpu.py"], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1500)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0 and "41 passed" in p.stdout and "skipped" not in p.stdout and "failed" not in p.stdout, \
        p.stdout[-3000:]
