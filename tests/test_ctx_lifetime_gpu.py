"""Closing a context gives back every device buffer it allocated.  Six create / use / close cycles run in a child
process (ctx_lifetime_child.py), each touching every kind of buffer a context holds; free device memory after the
last cycle must be within LEAK_LIMIT of free memory after the first.  A context that kept its 1M-offer table's
bit-sliced views would lose about 82 MiB per cycle.  Free memory is device-wide, so other work on the same GPU moves
it too: the limit leaves room for that."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
CHILD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ctx_lifetime_child.py")
LEAK_LIMIT = 64 << 20


def test_close_frees_device_memory():
    env = dict(os.environ)
    env.pop("RPK_FORCE_KERNEL", None)
    env.pop("RPK_TUNE", None)
    out = subprocess.run([sys.executable, CHILD], env=env, capture_output=True, text=True, timeout=1200)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-4000:]
    lines = out.stdout.strip().splitlines()
    assert lines[-1] == "ok", out.stdout[-4000:]
    free = json.loads(lines[-2])["free_bytes"]
    drop = free[0] - free[-1]
    per_cycle = ", ".join(f"{f / 2**20:.0f}" for f in free)
    assert drop < LEAK_LIMIT, f"free device memory fell by {drop / 2**20:.1f} MiB from cycle 1 to cycle {len(free)} " \
                              f"(MiB free after each cycle: {per_cycle})"
