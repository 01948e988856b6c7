"""tests/cpp/host_values_replay_test.cpp: the Go storage adaptor's call sequence with Config.HostValues (open with
KB_CFG_HOST_VALUES, load, List, commit batches, dump, restore into the other placement), compiled here against the
in-tree library and checked against the same calls in device placement."""
from __future__ import annotations

import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_host_values_replay_cpp(tmp_path):
    gxx = shutil.which("g++")
    assert gxx, "the replay driver needs a C++ compiler"
    libdir = os.path.join(ROOT, "kubebrain_b200")
    exe = str(tmp_path / "host_values_replay_test")
    subprocess.check_call([gxx, "-O1", "-std=c++17", "-Wall", "-o", exe,
                           os.path.join(ROOT, "tests", "cpp", "host_values_replay_test.cpp"),
                           "-L" + libdir, "-lkbb200", "-Wl,-rpath," + libdir])
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "host values replay ok" in r.stdout, r.stdout + r.stderr
