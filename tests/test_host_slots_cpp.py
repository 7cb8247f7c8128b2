"""Runs host/host_slots_test.cc: the Provider's sweep diffs only the slots it fetched (rpk_status_diff_slots), so the
engine's status_records grows by the fetched pods, not by the tracked table."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "host")
BIN = os.path.join(HOST, "host_slots_test")


@pytest.mark.gpu
def test_sweep_diffs_fetched_slots_only():
    if not os.path.exists(BIN):
        subprocess.check_call(["make", "-C", HOST, "-s"])
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1].startswith("ok:") and "0 failed" in out.stdout
