"""Builds and runs the C++ host-mirror test (tests/cpp/test_host.cpp) against libfamsa_b200.so."""
import subprocess

import pytest

from cpp_build import build_cpp


def test_host_mirror_compiles(tmp_path):
    build_cpp("test_host", tmp_path, famsa=True, oracle=True)


@pytest.mark.gpu
def test_host_mirror_runs(tmp_path):
    out = subprocess.run([build_cpp("test_host", tmp_path, famsa=True, oracle=True)], capture_output=True, text=True)
    assert out.returncode == 0 and "host mirror ok" in out.stdout, out.stdout + out.stderr
