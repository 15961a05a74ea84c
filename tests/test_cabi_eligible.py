"""The C driver of node eligibility (tests/cabi_eligible.c): rbgtopo_set_node_classes and
rbgtopo_place_groups_eligible[_ranked] called the way the cgo shim's helpers call them — the call and the error fetch on
one OS thread, a sequential repeat, ten placing OS threads on one ctx beside one that re-installs the classes and the
capacities, and every error code."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rbg_b200", "csrc")


def _build(tmp_path):
    exe = str(tmp_path / "cabi_eligible")
    subprocess.run(["gcc", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cabi_eligible.c"), "-L" + CSRC,
                    "-lrbgtopo", "-lpthread", "-Wl,-rpath," + CSRC], check=True, capture_output=True, text=True)
    return exe


def test_cabi_eligible_host(tmp_path):
    r = subprocess.run([_build(tmp_path), "host"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "CABI_ELIGIBLE_OK host" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_cabi_eligible_gpu(tmp_path):
    r = subprocess.run([_build(tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "CABI_ELIGIBLE_OK gpu" in r.stdout, r.stdout + r.stderr
