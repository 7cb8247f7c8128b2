"""Runs host/host_pods_test.cc: the Provider's pending-pod tick seeds only the pod-table rows whose columns changed and
selects by slot (rpk_select_slots); a changed pod or owner-Job annotation and a reused slot reach the selection, and a
random population gets the gpuTypeIds PrepareColumnsBatch + rpk_select give it."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "host")
BIN = os.path.join(HOST, "host_pods_test")


@pytest.mark.gpu
def test_pending_tick_seeds_changed_rows_and_selects_by_slot():
    if not os.path.exists(BIN):
        subprocess.check_call(["make", "-C", HOST, "-s"])
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1].startswith("ok:") and "0 failed" in out.stdout
