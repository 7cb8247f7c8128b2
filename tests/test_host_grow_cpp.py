"""Runs host/host_grow_test.cc: a Provider that starts at 16 slots grows its pod and status tables in place as pods
arrive, instead of refusing the pod past its capacity; 5 000 pods over many ticks and sweeps deploy and notify exactly as
on a Provider built with 8 192 slots, and concurrent creates, deletes and sweeps across several growths lose no
notification."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "host")
BIN = os.path.join(HOST, "host_grow_test")


@pytest.mark.gpu
def test_provider_grows_past_its_initial_capacity():
    if not os.path.exists(BIN):
        subprocess.check_call(["make", "-C", HOST, "-s"])
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1].startswith("ok:") and "0 failed" in out.stdout
