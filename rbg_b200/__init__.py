"""rbg_b200 — H100-native topology-aware placement hot path for sgl-project/rbg.

Only what the path needs lives here (DESIGN.md §1):
  csrc/      sm_90a CUDA kernels + the C-ABI runtime (librbgtopo.so, include/rbgtopo.h)
  _lib.py    ctypes binding of the C ABI (fails loudly when the .so is missing)
  engine.py  thin object wrapper over a rbgtopo_ctx
  blob.py    builder of the batch wire format
  plugin.py  host-side mirror of the reference plugin surface
             (scheduler.PodGroupManager, pkg/scheduler/podgroup_manager.go:64-78)
  synth.py   seeded synthetic topologies / RBG fleets (SURVEY.md §8d)
There is no CPU fallback anywhere in this package.
"""
from .blob import BlobBuilder, Step  # noqa: F401


def __getattr__(name):   # engine (and with it the ctypes binding) only when somebody asks for it:
    if name in ("TopoPlacer", "RbgTopoError"):   # `import rbg_b200.synth` must stay free of native code
        from . import engine
        return getattr(engine, name)
    raise AttributeError(name)
