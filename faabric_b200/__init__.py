"""faabric_b200 — a Hopper (H100, sm_90a) native distributed runtime with
the capabilities of faasm/faabric: Planner / Scheduler / Executor, MpiWorld,
PointToPointBroker, SnapshotRegistry, StateKeyValue — with ranks bound to GPUs
and the communication-bound hot paths implemented as hand-written CUDA kernels
that read and write peer HBM over NVLink / NVSwitch.

Layout:
  faabric_b200.parallel  communicators, symmetric heap, process-group bootstrap
  faabric_b200.ops       collectives / snapshot / state device ops
  faabric_b200.models    workload definitions (ResNet-50 gradient sync, ...)
  faabric_b200.utils     timing, clocks sampling, roofline helpers
  faabric_b200.runtime   bindings to the native C++ runtime (planner, MPI, ...)
"""

__version__ = "0.1.0"

import os as _os

# CUDA maps streams onto a limited number of hardware work queues (8 by
# default).  Streams that share a queue serialise: a stream-level wait (or a
# kernel polling a flag) of one rank can then sit in front of the very signal
# kernel of another rank it is waiting for.  Several ranks per GPU times several
# lanes per rank needs more queues than the default; the variable is only read
# when the CUDA context is created, so it has to be in place at import time.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from . import _lib  # noqa: F401


def native_library_path():
    return _lib.lib_path()
