"""Builds librsp_b200.so (CUDA kernels + engine + C ABI) in-tree with nvcc for sm_90a (H100).

    python -m rocksplicator_b200.build [--force]

The .so and the objects under build/ are git-ignored build products.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "librsp_b200.so")
SOURCES = ["k_apply.cu", "k_read.cu", "k_compact.cu", "engine.cu"]
HEADERS = ["format.cuh", "kernels.h", "stager.h", "arena.h", "reader_set.h", os.path.join("..", "..", "include", "rsp_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall"] + os.environ.get("RSP_NVCC_EXTRA", "").split()


def _nvcc():
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + hdrs):
            jobs.append([_nvcc()] + NVCC_FLAGS + ["-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)

    with ThreadPoolExecutor(max_workers=4) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(objdir, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(OUT, objs):
        run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-o", OUT] + objs +
            ["-cudart", "static", "-lpthread", "-ldl", "-lrt"])
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))


HOST = os.path.join(HERE, "host")
HOST_SRCS = ["gpu_db.cpp", "rocksdb_replicator/rocksdb_replicator.cpp", "rocksdb_replicator/gpu_db_wrapper.cpp",
             "rocksdb_admin/application_db.cpp", "rocksdb_admin/application_db_manager.cpp", "sst/sst_c_api.cpp",
             "bench/seam_bench.cpp", "rocksdb_admin/message_ingestion.cpp"]
HOST_SO = os.path.join(HERE, "librsp_host.so")
HOST_TESTS = os.path.join(os.path.dirname(HERE), "tests", "cpp", "host_tests")
SNAPSHOT_TESTS = os.path.join(os.path.dirname(HERE), "tests", "cpp", "snapshot_tests")
BOUNDED_ITER_TESTS = os.path.join(os.path.dirname(HERE), "tests", "cpp", "bounded_iter_tests")
STRING_APPEND_TESTS = os.path.join(os.path.dirname(HERE), "tests", "cpp", "string_append_tests")
INGEST_BEHIND_TESTS = os.path.join(os.path.dirname(HERE), "tests", "cpp", "ingest_behind_tests")


def build_host(force=False, verbose=False):
    """The C++ mirror of the reference interfaces (host/) -> librsp_host.so, and its test binaries (snapshot_tests,
    bounded_iter_tests, string_append_tests and ingest_behind_tests are returned by build_snapshot_tests,
    build_bounded_iter_tests, build_string_append_tests and build_ingest_behind_tests)."""
    build(force=False, verbose=verbose)
    srcs = [os.path.join(HOST, s) for s in HOST_SRCS]
    deps = list(srcs)
    for dp, _, fs in os.walk(HOST):
        deps += [os.path.join(dp, f) for f in fs if f.endswith(".h")]
    cxx = os.environ.get("CXX", "g++")
    flags = ["-std=c++17", "-O2", "-g", "-fPIC", "-Wall", "-I", HOST, "-pthread"]

    def run(cmd):
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)

    if force or _stale(HOST_SO, deps + [OUT]):
        run([cxx] + flags + ["-shared", "-o", HOST_SO] + srcs + ["-L", HERE, "-lrsp_b200", "-Wl,-rpath,$ORIGIN"])
    tsrc = os.path.join(os.path.dirname(HERE), "tests", "cpp", "host_tests.cpp")
    if force or _stale(HOST_TESTS, [tsrc, HOST_SO] + deps):
        run([cxx] + flags + ["-o", HOST_TESTS, tsrc, "-L", HERE, "-lrsp_host", "-lrsp_b200",
                             "-Wl,-rpath," + HERE])
    for exe in (SNAPSHOT_TESTS, BOUNDED_ITER_TESTS, STRING_APPEND_TESTS, INGEST_BEHIND_TESTS):
        src = exe + ".cpp"
        if force or _stale(exe, [src, HOST_SO] + deps):
            run([cxx] + flags + ["-o", exe, src, "-L", HERE, "-lrsp_host", "-lrsp_b200", "-Wl,-rpath," + HERE])
    return HOST_SO, HOST_TESTS


def build_snapshot_tests(force=False, verbose=False):
    """tests/cpp/snapshot_tests: GpuDB / ApplicationDB reads with ReadOptions::snapshot"""
    build_host(force=force, verbose=verbose)
    return SNAPSHOT_TESTS


def build_bounded_iter_tests(force=False, verbose=False):
    """tests/cpp/bounded_iter_tests: GpuDB / ApplicationDB iterators with ReadOptions::iterate_upper_bound and
    SeekForPrev"""
    build_host(force=force, verbose=verbose)
    return BOUNDED_ITER_TESTS


def build_string_append_tests(force=False, verbose=False):
    """tests/cpp/string_append_tests: rocksdb::StringAppendOperator through GpuDB / ApplicationDB (the device operator,
    reads at snapshots, Backup / Restore)"""
    build_host(force=force, verbose=verbose)
    return STRING_APPEND_TESTS


def build_ingest_behind_tests(force=False, verbose=False):
    """tests/cpp/ingest_behind_tests: Options::allow_ingest_behind, IngestExternalFileOptions::ingest_behind and
    CompactRange(change_level) through GpuDB / ApplicationDB (application_db_test.cpp:300-342 step for step)"""
    build_host(force=force, verbose=verbose)
    return INGEST_BEHIND_TESTS
