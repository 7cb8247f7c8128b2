"""Runs host/host_pending_test.cc: the Provider's pending-pod tick uploads only the pending flags that changed and
selects with rpk_select_pending, without a slot list; deployed, deleted and failed pods leave the set, a reused slot is
marked again, a pod created or deployed elsewhere during a tick is neither lost nor deployed twice, and a random
population with churn gets the gpuTypeIds PrepareColumnsBatch + rpk_select give it."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "host")
BIN = os.path.join(HOST, "host_pending_test")


@pytest.mark.gpu
def test_pending_tick_marks_changed_flags_and_selects_the_pending_set():
    if not os.path.exists(BIN):
        subprocess.check_call(["make", "-C", HOST, "-s"])
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1].startswith("ok:") and "0 failed" in out.stdout
