"""Builds and runs the C++ host mirror's passes::IqWatch (include/noaa_apt.hpp) against libaptb200.so."""
import os
import subprocess

import pytest

import __graft_entry__ as entry

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(tmp_path):
    entry.build()
    exe = str(tmp_path / "watch_iq_mirror")
    libdir = os.path.join(ROOT, "noaa-apt_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "watch_iq_mirror.cpp"), "-o", exe,
                           "-L", libdir, "-laptb200", f"-Wl,-rpath,{libdir}"])
    return exe


def test_cpp_watch_iq_host_logic(tmp_path):
    out = subprocess.run([_build(tmp_path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "OK host" in out.stdout


@pytest.mark.gpu
def test_cpp_watch_iq_equals_a_watch_per_channel(tmp_path):
    out = subprocess.run([_build(tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "OK gpu" in out.stdout
