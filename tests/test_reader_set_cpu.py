"""csrc/reader_set.h alone (std only, fake streams and events): which reads on callers' streams a flush, merge install,
snapshot pin or shard close waits for.  The CPU emulation cannot check this, because its streams are synchronous."""
import os
import subprocess


def test_reader_set(tmp_path):
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "reader_set_test.cpp")
    cxx = os.environ.get("CXX", "g++")
    exe = str(tmp_path / "reader_set_test")
    flags = ["-std=c++17", "-O1", "-g", "-Wall"]
    if subprocess.call([cxx] + flags + ["-fsanitize=address", src, "-o", exe], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL) != 0:
        subprocess.check_call([cxx] + flags + [src, "-o", exe])
    p = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(p.stdout, p.stderr[-2000:])
    assert p.returncode == 0 and "bad 0" in p.stdout
