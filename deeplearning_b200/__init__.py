"""deeplearning_b200: an H100-native (sm_90a) implementation of the KKKSQJ/DeepLearning classification training step.

Layout
  csrc/            hand-written CUDA (wgmma / TMA / mbarrier) + the C-ABI (include/b200cls.h) -> lib/libb200cls.so
  _lib.py, ops.py  ctypes binding and tensor-level wrappers (PyTorch = device memory + streams only)
  engine/          forward/backward schedules of the backbones, gradient arena + data-parallel step
  classification/  host-side mirrors of the reference constructors (same names, signatures, state_dict keys)
"""
__version__ = "0.1.0"
