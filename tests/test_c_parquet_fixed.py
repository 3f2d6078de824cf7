"""tests/c/pq_fixed_smoke.c, a plain-C program calling ag_parquet_bool_decode and ag_parquet_fixed_decode, compiled with
gcc against include/arrowgpu.h and linked with libarrowgpu.so.  Without a GPU it must build, link and be refused (both
calls, output untouched); on the GPU it must pass its own checks."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(tmp):
    exe = os.path.join(tmp, "pq_fixed_smoke")
    lib = os.path.join(ROOT, "arrow_go_b200", "lib")
    cmd = ["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c", "pq_fixed_smoke.c"), "-o", exe, "-L", lib, "-larrowgpu", f"-Wl,-rpath,{lib}"]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return exe


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_fixed_c_program_builds_and_is_refused_without_gpu(tmp_path):
    out = subprocess.run([build(str(tmp_path))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 77, (out.returncode, out.stdout, out.stderr)


@pytest.mark.gpu
def test_fixed_c_program_on_gpu(tmp_path):
    out = subprocess.run([build(str(tmp_path))], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert "pq_fixed_smoke ok" in out.stdout
