"""rsp::ArenaBlock, the owning handle of one block of csrc/arena.h (tests/cpp/arena_block_test.cpp), over malloc under
AddressSanitizer: destruction releases, a move hands the block on, move-assignment releases the target's block, an
empty handle releases nothing, and the arena's invariants hold throughout"""
import os
import subprocess


def test_arena_block_handle(tmp_path):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "arena_block_test.cpp")
    cxx = os.environ.get("CXX", "g++")
    exe = str(tmp_path / "arena_block_test")
    flags = ["-std=c++17", "-O1", "-g", "-pthread"]
    if subprocess.call([cxx] + flags + ["-fsanitize=address", src, "-o", exe], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL) != 0:
        subprocess.check_call([cxx] + flags + [src, "-o", exe])
    p = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(p.stdout, p.stderr[-2000:])
    assert p.returncode == 0 and "bad 0" in p.stdout
