"""easydist_b200 — H100-native (sm_90a) SPMD execution backend for the easydist.torch hot path.

What lives here is only what the path needs (SURVEY.md §8):
  csrc/ + include/edb.h   CUDA kernels behind a C-ABI (libedb.so)
  _lib / runtime          ctypes binding, symmetric heap + peer mapping bootstrap
  reshard                 the reference's ten reshard callables, same names/semantics
  gemm                    sharded-op kernel dispatch (wgmma GEMM)
  metair / planners       plan vocabulary + edge planners (mirror of metair.py / sharding.py)
  lowering                sharding_transform / transform_ddp / transform_fsdp replacements
  compile / api           tracing front-end, executor, `easydist_compile` entry point
"""
__version__ = "0.1.0"
