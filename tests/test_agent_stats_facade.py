"""Per-agent Stats() through the C++ serf facade (tests/facade/agent_stats_check.cpp).  CPU: linked with the host
emulation; GPU: with libgsim.so."""
import os
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "facade", "agent_stats_check.cpp")


def build_and_run(libdir, libname):
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "agent_stats_check")
        subprocess.run(["g++", "-O1", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-o", out, SRC,
                        "-L" + libdir, "-l" + libname, "-Wl,-rpath," + libdir], check=True, cwd=ROOT)
        r = subprocess.run([out], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    for name in ("PASS Serf.Stats per agent", "ALL PASS"):
        assert name in r.stdout, r.stdout


def test_agent_stats_facade_on_host_emulation():
    build_and_run(os.path.join(ROOT, "tests", "hostemu"), "gsim_hostemu")


@pytest.mark.gpu
def test_agent_stats_facade_on_cuda():
    build_and_run(os.path.join(ROOT, "consul_b200"), "gsim")
