"""rpk -- H100-native batch scheduling engine for the RunPod virtual kubelet's hot path.

The directory name carries the reference's name and is not a valid Python identifier; import it with
``importlib.import_module("k8s-runpod-kubelet_b200")`` (see ``__graft_entry__.py``) or through the ``rpk``
alias module at the repo root.

Contents: ``csrc/`` (CUDA kernels + the C-ABI of ``include/rpk.h``), ``lib/librpk.so`` (built in-tree),
``_ffi`` / ``engine`` (ctypes binding, the same ABI a cgo binding calls), ``synth`` (deterministic tables),
``host/`` (C++ mirror of the reference's Provider surface for this path).
"""
from . import _ffi, synth  # noqa: F401
from .engine import Engine, results_region  # noqa: F401
from ._ffi import RpkError  # noqa: F401

__all__ = ["Engine", "RpkError", "results_region", "synth"]
