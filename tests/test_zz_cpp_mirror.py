"""The C++ mirror of the reference's front door (liquid_cache_b200/csrc/liquid_cache.hpp: LiquidCacheBuilder, insert / get /
eval_predicate builders, LiquidExpr) driven by a C++ program that replays the reference's quick-start examples
(/root/reference/README.md:43-88, src/core/README.md:17-104) — tests/cpp/quickstart.cc, compiled with g++ against
include/lc_gpu.h and the in-tree liblc_gpu.so. Without a CUDA device the program must stop at the first call with the
library's "no CPU fallback" error (exit code 3); on an H100 every published answer must come out (exit code 0)."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_DIR = os.path.join(ROOT, "liquid_cache_b200", "lib")
EXE = os.path.join(ROOT, "build", "tests", "quickstart")


def _build():
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT}", os.path.join(ROOT, "tests", "cpp", "quickstart.cc"), "-o", EXE,
           f"-L{LIB_DIR}", "-llc_gpu", f"-Wl,-rpath,{LIB_DIR}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return subprocess.run([EXE], capture_output=True, text=True, timeout=300)


def test_cpp_mirror_compiles_and_refuses_to_run_without_a_device():
    r = _build()
    assert r.returncode in (0, 3), (r.returncode, r.stdout, r.stderr)
    if r.returncode == 3:
        assert "no device" in r.stderr and "no CPU fallback" in r.stderr, r.stderr


@pytest.mark.gpu
def test_cpp_mirror_reproduces_the_quick_start_answers():
    r = _build()
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "0 wrong answers" in r.stdout, r.stdout
