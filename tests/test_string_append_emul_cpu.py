"""CPU-only: tests/test_string_append_gpu.py against the CPU emulation build of the engine (tests/emul/build_emul.py), in
a subprocess, as tests/test_snapshot_scan_emul_cpu.py does for the scans at snapshots; and a seeded differential of
random streams (every delimiter, random flush and compaction points) between the emulated engine and the model of
tests/string_append_model.py.  This catches logic and addressing bugs of the string-append fold before GPU time is
spent; the `-m gpu` run on an H100 is the real test."""
import importlib.util
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _emul_env():
    spec = importlib.util.spec_from_file_location("build_emul", os.path.join(ROOT, "tests", "emul", "build_emul.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib = mod.build()[0]
    env = dict(os.environ)
    env["RSP_TEST_EMUL_LIB"] = lib
    env.setdefault("RSP_TEST_EMUL_ARENA", str(16 << 20))
    return env


def test_string_append_suite_under_emulation():
    p = subprocess.run([sys.executable, "-m", "pytest", "-m", "gpu", "-x", "-q", "-p", "no:cacheprovider",
                        "tests/test_string_append_gpu.py"], cwd=ROOT, env=_emul_env(), capture_output=True, text=True,
                       timeout=1500)
    print(p.stdout[-3000:], p.stderr[-2000:])
    assert p.returncode == 0 and " passed" in p.stdout and "failed" not in p.stdout, p.stdout[-3000:]


_DIFFERENTIAL = r'''
import os, random, sys
sys.path.insert(0, "tests")
import string_append_model as SA
from rocksplicator_b200 import engine
engine.SO_PATH = os.environ["RSP_TEST_EMUL_LIB"]
e = engine.Engine(0, arena_bytes=int(os.environ["RSP_TEST_EMUL_ARENA"]), l0_compaction_trigger=3)
n_streams = int(sys.argv[1])
for seed in range(n_streams):
    rng = random.Random(seed)
    delim = [b",", None, b"\0", b"|"][seed % 4]
    s = e.open_shard("diff%d" % seed, merge_op=engine.MERGE_STRING_APPEND, merge_delim=delim)
    m = SA.Model(delim)
    keys = [b"k%d" % i for i in range(rng.choice([3, 8, 20]))]
    for step in range(rng.randrange(4, 12)):
        ops = []
        for _ in range(rng.randrange(1, 8)):
            k, r = rng.choice(keys), rng.random()
            if r < 0.6:
                ops.append((SA.MERGE, k, bytes(rng.randrange(97, 100) for _ in range(rng.randrange(0, 5)))))
            elif r < 0.8:
                ops.append((SA.PUT, k, b"" if rng.random() < 0.3 else b"P%d" % step))
            else:
                ops.append((SA.DEL, k, b""))
        assert s.apply(SA.batch_of(ops), 0) == 0
        m.apply(ops)
        r = rng.random()
        if r < 0.3:
            assert s.flush() == 0
        elif r < 0.4:
            assert s.compact() == 0
        got = s.multi_get(keys, stride=4)
        want = [(0, m.get(k)) if m.get(k) is not None else (1, None) for k in keys]
        assert got == want, (seed, step, got, want)
        assert s.scan() == m.items(), (seed, step)
    s.close()
print("streams", n_streams)
'''


def test_random_streams_against_the_model_under_emulation():
    p = subprocess.run([sys.executable, "-c", _DIFFERENTIAL, "300"], cwd=ROOT, env=_emul_env(), capture_output=True,
                       text=True, timeout=1500)
    print(p.stdout[-3000:], p.stderr[-3000:])
    assert p.returncode == 0 and "streams 300" in p.stdout, p.stderr[-3000:]
