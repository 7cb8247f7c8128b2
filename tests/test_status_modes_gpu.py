"""GPU tests of the big-table streaming loop modes of the status sweep (DESIGN §4: units, beats, beats4 and ring give
the same results).  The mode is read once per process (RPK_TUNE k2=...), so each runs in a child process
(tests/status_mode_child.py) over the big-table boundary at strides 16 and 32, host and device entry points."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
CHILD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "status_mode_child.py")


@pytest.mark.parametrize("mode", ["units", "beats", "beats4", "ring"])
def test_big_table_loop_mode(mode):
    env = dict(os.environ, RPK_TUNE=f"k2={mode}")
    out = subprocess.run([sys.executable, CHILD], env=env, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-4000:] + out.stderr[-4000:]
    assert out.stdout.strip().splitlines()[-1] == f"ok k2={mode}"
