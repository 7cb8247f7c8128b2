"""Runs host/host_explain_test.cc: Provider::ExplainUnschedulable lists exactly the pending pods whose gpuTypeIds list
came back empty, with the pinned scheduler-style messages on the ten offers of SURVEY.md 8(c); a pod whose annotation is
fixed drops out after the next tick; the deploys and notifications equal those of a Provider that never calls it; and
on a random mix every explanation equals rpk_explain of the pod's columns."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "k8s-runpod-kubelet_b200", "host")
BIN = os.path.join(HOST, "host_explain_test")


@pytest.mark.gpu
def test_provider_explains_unschedulable_pods():
    if not os.path.exists(BIN):
        subprocess.check_call(["make", "-C", HOST, "-s"])
    out = subprocess.run([BIN], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-2000:]
    assert out.stdout.strip().splitlines()[-1].startswith("ok:") and "0 failed" in out.stdout
