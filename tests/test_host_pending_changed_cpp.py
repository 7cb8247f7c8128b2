"""Runs host/host_pending_changed_test.cc: the Provider's pending tick with rpk_select_pending_changed deploys every
pending pod from its per-slot mirror of top-5 lists with the gpuTypeIds a reference select gives; a steady tick
recomputes no row, a one-price offer refresh changes only the affected pods' lists, and a reused slot with identical
columns deploys with the right ids."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "host")
BIN = os.path.join(HOST, "host_pending_changed_test")


@pytest.mark.gpu
def test_pending_tick_deploys_from_the_mirror_of_changed_lists():
    if not os.path.exists(BIN):
        subprocess.check_call(["make", "-C", HOST, "-s"])
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1].startswith("ok:") and "0 failed" in out.stdout
