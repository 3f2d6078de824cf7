"""The plain-C programs under tests/c, each compiled with gcc against include/arrowgpu.h and linked with libarrowgpu.so:
the boundary is a C ABI any FFI can bind.  Without a GPU each must build, link, run and be refused by the library (no
CPU fallback); on the GPU each must pass its own checks."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (program, the line it prints when its checks pass)
PROGRAMS = [
    ("abi_smoke", "abi_smoke ok"),                  # device count, reductions, the error text
    ("pq_smoke", "pq_smoke ok"),                    # ag_parquet_dict_decode
    ("pq_delta_smoke", "pq_delta_smoke ok"),        # ag_parquet_delta_decode
    ("pq_snappy_smoke", "pq_snappy_smoke ok"),      # ag_parquet_snappy_decompress
    ("pq_zstd_smoke", "pq_zstd_smoke ok"),          # ag_parquet_zstd_decompress
    ("pq_gzip_smoke", "pq_gzip_smoke ok"),          # ag_parquet_gzip_decompress
    ("pq_lz4_smoke", "pq_lz4_smoke ok"),            # ag_parquet_lz4_raw_decompress
    ("pq_bytearray_smoke", "pq_bytearray_smoke ok"),  # ag_parquet_byte_array_decode
    ("pq_fixed_smoke", "pq_fixed_smoke ok"),        # ag_parquet_bool_decode and ag_parquet_fixed_decode
]
EACH = pytest.mark.parametrize("name,ok", PROGRAMS, ids=[p[0] for p in PROGRAMS])


def build(name, tmp):
    exe = os.path.join(tmp, name)
    lib = os.path.join(ROOT, "arrow_go_b200", "lib")
    cmd = ["gcc", "-std=c11", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "c", name + ".c"), "-o", exe, "-L", lib, "-larrowgpu", f"-Wl,-rpath,{lib}"]
    out = subprocess.run(cmd, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return exe


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
@EACH
def test_c_program_builds_and_is_refused_without_gpu(name, ok, tmp_path):
    out = subprocess.run([build(name, str(tmp_path))], capture_output=True, text=True, timeout=120)
    assert out.returncode == 77, (out.returncode, out.stdout, out.stderr)
    if name == "abi_smoke":
        assert "no CPU fallback" in out.stdout


@pytest.mark.gpu
@EACH
def test_c_program_on_gpu(name, ok, tmp_path):
    out = subprocess.run([build(name, str(tmp_path))], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, (out.returncode, out.stdout, out.stderr)
    assert ok in out.stdout
