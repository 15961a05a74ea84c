"""The C driver of node eligibility in committed batches (tests/cabi_eligible_committed.c):
rbgtopo_place_groups_eligible_committed[_ranked] called the way the cgo shim's helpers call them — the call and the
error fetch on one OS thread, a sequential repeat, ten OS threads making both calls on one ctx beside one that
re-installs the classes and the capacities, and the error codes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rbg_b200", "csrc")


def _build(tmp_path):
    exe = str(tmp_path / "cabi_eligible_committed")
    subprocess.run(["gcc", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cabi_eligible_committed.c"),
                    "-L" + CSRC, "-lrbgtopo", "-lpthread", "-Wl,-rpath," + CSRC], check=True, capture_output=True,
                   text=True)
    return exe


def test_cabi_eligible_committed_host(tmp_path):
    r = subprocess.run([_build(tmp_path), "host"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "CABI_ELIGIBLE_COMMITTED_OK host" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_cabi_eligible_committed_gpu(tmp_path):
    r = subprocess.run([_build(tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "CABI_ELIGIBLE_COMMITTED_OK gpu" in r.stdout, r.stdout + r.stderr
