"""CPU-only: tests/test_ingest_behind_gpu.py against the CPU emulation build of the engine (tests/emul/build_emul.py), in
a subprocess, as tests/test_scan_boundaries_emul_cpu.py does for its suite.  This runs the ingest-behind refusals, the
tier's path through flushes and compactions, the device-built ingest runs at their size boundaries and the seeded
random differential against the oracle port ("the behind files first") without a GPU; the emulation enforces neither
the shared-memory limits nor the warp-level ordering of the hardware, so the `-m gpu` run on an H100 is the real test."""
import importlib.util
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ingest_behind_suite_under_emulation():
    spec = importlib.util.spec_from_file_location("build_emul", os.path.join(ROOT, "tests", "emul", "build_emul.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib = mod.build()[0]
    env = dict(os.environ)
    env["RSP_TEST_EMUL_LIB"] = lib
    env.setdefault("RSP_TEST_EMUL_ARENA", str(16 << 20))
    p = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider",
                        "tests/test_ingest_behind_gpu.py"], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1500)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-3000:]
