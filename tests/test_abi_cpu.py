"""CPU-only: the C-ABI library builds, loads and exports every symbol include/rsp_b200.h declares."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from rocksplicator_b200 import build, engine
    build.build()
    return engine.load_library()


def test_every_declared_symbol_is_exported(lib):
    from rocksplicator_b200 import engine
    hdr = open(os.path.join(ROOT, "include", "rsp_b200.h")).read()
    declared = set(re.findall(r"\b(rsp_[a-z0-9_]+)\s*\(", hdr)) - {"rsp_merge_fn"}
    assert declared, "no declarations parsed"
    missing_in_binding = declared - set(engine.EXPORTS)
    assert not missing_in_binding, missing_in_binding
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.rsp_version().startswith(b"rocksplicator_b200")


def test_no_cpu_fallback_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from rocksplicator_b200 import engine
    with pytest.raises(RuntimeError):
        engine.Engine(0)


def test_product_does_not_touch_oracle():
    pkg = os.path.join(ROOT, "rocksplicator_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".cc")):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert "okv_" not in txt and "import oracle" not in txt and "from oracle" not in txt, f


def test_product_library_has_no_emulation_or_cpu_path():
    """librsp_b200.so is the nvcc build: none of tests/emul's symbols, device code for sm_90a inside, and the Python
    binding names no other library.  (tests/emul builds a separate test-only library from the same sources.)"""
    import subprocess
    from rocksplicator_b200 import engine
    so = os.path.join(ROOT, "rocksplicator_b200", "librsp_b200.so")
    assert os.path.realpath(engine.SO_PATH) == os.path.realpath(so)
    syms = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True, check=True).stdout
    assert "emul_launch" not in syms and "emul_collective" not in syms
    elf = subprocess.run(["cuobjdump", "-lelf", so], capture_output=True, text=True)
    if elf.returncode == 0:  # cuobjdump ships with the CUDA toolkit
        assert "sm_90a" in elf.stdout, elf.stdout[:300]
    for dp, _, fs in os.walk(os.path.join(ROOT, "rocksplicator_b200")):
        for f in fs:
            if f.endswith(".py"):
                txt = open(os.path.join(dp, f), errors="ignore").read()
                assert "tests/emul" not in txt and "_emul.so" not in txt and "RSP_TEST_EMUL" not in txt, f
