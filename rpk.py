"""Importable alias for the package directory ``k8s-runpod-kubelet_b200`` (not a valid identifier)."""
import importlib
import os
import sys

_ROOT = os.path.dirname(os.path.abspath(__file__))
if _ROOT not in sys.path:
    sys.path.insert(0, _ROOT)
_pkg = importlib.import_module("k8s-runpod-kubelet_b200")
Engine = _pkg.Engine
RpkError = _pkg.RpkError
results_region = _pkg.results_region
synth = _pkg.synth
_ffi = _pkg._ffi
