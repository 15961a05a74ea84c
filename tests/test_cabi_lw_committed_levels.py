"""The C driver of committed leader-worker batches at exclusive levels (tests/cabi_lw_committed_levels.c):
rbgtopo_place_groups_lw_committed and its ranked form on a ctx with RBGTOPO_CFG_LW_COMMIT_LEVELS, called the way the
cgo shim calls them — the call and the error fetch on one OS thread, a sequential repeat and ten OS threads on one
ctx."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rbg_b200", "csrc")


def _build(tmp_path):
    exe = str(tmp_path / "cabi_lw_committed_levels")
    subprocess.run(["gcc", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cabi_lw_committed_levels.c"), "-L" + CSRC,
                    "-lrbgtopo", "-lpthread", "-Wl,-rpath," + CSRC], check=True, capture_output=True, text=True)
    return exe


def test_cabi_lw_committed_levels_host(tmp_path):
    r = subprocess.run([_build(tmp_path), "host"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "CABI_LW_COMMITTED_LEVELS_OK host" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_cabi_lw_committed_levels_gpu(tmp_path):
    r = subprocess.run([_build(tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "CABI_LW_COMMITTED_LEVELS_OK gpu" in r.stdout, r.stdout + r.stderr
