"""cdprobe — H100-native ComputeDomain fabric-validation probe.

The product is ``libcdprobe.so`` (hand-written sm_90a CUDA + a C++ host
runtime behind the C ABI in ``include/cdprobe.h``).  This package is the thin
host-side mirror of the Go shim ``pkg/fabricprobe`` a maintainer would add to
NVIDIA/k8s-dra-driver-gpu (SURVEY.md §8b, INTEGRATION.md): same names, same
argument meaning, same error behaviour, bound with ctypes instead of cgo because
this image has no Go toolchain.

The directory name contains hyphens (the layout the task prescribes); import it
through ``cdprobe_pkg.load()`` at the repo root, which registers it as
``k8s_dra_driver_gpu_b200``.
"""
from . import abi, build, distutil  # noqa: F401
from .fabricprobe import (  # noqa: F401
    AllReduce,
    Atomics,
    BwCurve,
    Config,
    Diagnosis,
    ErrUnsupported,
    Latency,
    PingPong,
    Probe,
    ProbeError,
    Result,
    Open,
    gate,
    plan,
    topology,
)

__all__ = ["abi", "build", "Config", "Probe", "ProbeError", "ErrUnsupported", "Result", "Diagnosis", "Latency", "PingPong", "Atomics", "BwCurve", "AllReduce", "Open", "gate", "plan", "topology"]
