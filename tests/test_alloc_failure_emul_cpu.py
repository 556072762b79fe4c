"""tests/emul/alloc_failure_sweep.py against the AddressSanitizer build of the emulation: every device and pinned
allocation of every maintenance operation (shard open, a memtable re-size, flush, compaction, change-level compaction,
snapshot, iterators, both ingest forms, a pre-staged tick image, host-form MultiGet and scan) made to fail in turn.  Each
failed call answers an IO error and leaves the shards as they were, with no device memory gained; nothing is left once
the engine is destroyed.  (No GPU twin: a GPU shared with other work is not driven out of memory on purpose.)"""
import importlib.util
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _runtime_lib(name):
    out = subprocess.run(["/usr/bin/g++", "-print-file-name=" + name], capture_output=True, text=True).stdout.strip()
    return out if os.path.isabs(out) and os.path.exists(out) else None


def test_every_allocation_of_every_maintenance_operation_fails_cleanly(tmp_path):
    asan, stdcxx = _runtime_lib("libasan.so"), _runtime_lib("libstdc++.so")
    if not asan or not stdcxx:
        pytest.skip("the system compiler has no AddressSanitizer runtime")
    spec = importlib.util.spec_from_file_location("build_emul", os.path.join(ROOT, "tests", "emul", "build_emul.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    lib, _ = mod.build(asan=True)
    hook = str(tmp_path / "liballoc_fail_hook.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-w", "-pthread", "-I",
                           os.path.join(ROOT, "tests", "emul", "include"),
                           os.path.join(ROOT, "tests", "emul", "alloc_fail_hook.cpp"), "-o", hook, "-ldl"])
    env = dict(os.environ)
    # libstdc++ is preloaded with the runtime, so that ASan's interceptor finds __cxa_throw for the engine's exceptions;
    # the hook goes in front of the emulated library, whose allocation calls it takes over
    env.update({"RSP_TEST_EMUL_LIB": lib, "RSP_EMUL_EXACT_ALLOC": "1", "LD_PRELOAD": " ".join([asan, stdcxx, hook]),
                "ASAN_OPTIONS": "detect_leaks=0"})
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "emul", "alloc_failure_sweep.py")], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    print(p.stdout[-3000:], p.stderr[-3000:])
    assert p.returncode == 0 and "ALLOC FAILURE SWEEP OK" in p.stdout
