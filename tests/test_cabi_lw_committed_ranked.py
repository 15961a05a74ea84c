"""The C driver of ranked committed leader-worker batches (tests/cabi_lw_committed_ranked.c):
rbgtopo_place_groups_lw_committed_ranked called the way the cgo shim's rbgtopo_go_place_groups_lw_committed_ranked helper
calls it — the call and the error fetch on one OS thread, a sequential repeat, ten OS threads on one ctx, and equality
with rbgtopo_place_groups_lw_committed."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rbg_b200", "csrc")


def _build(tmp_path):
    exe = str(tmp_path / "cabi_lw_committed_ranked")
    subprocess.run(["gcc", "-O1", "-Wall", "-o", exe, os.path.join(ROOT, "tests", "cabi_lw_committed_ranked.c"), "-L" + CSRC,
                    "-lrbgtopo", "-lpthread", "-Wl,-rpath," + CSRC], check=True, capture_output=True, text=True)
    return exe


def test_cabi_lw_committed_ranked_host(tmp_path):
    r = subprocess.run([_build(tmp_path), "host"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "CABI_LW_COMMITTED_RANKED_OK host" in r.stdout, r.stdout + r.stderr


@pytest.mark.gpu
def test_cabi_lw_committed_ranked_gpu(tmp_path):
    r = subprocess.run([_build(tmp_path), "gpu"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "CABI_LW_COMMITTED_RANKED_OK gpu" in r.stdout, r.stdout + r.stderr
