"""faer-rs_b200: H100-native (sm_90a) backend for faer's dense hot path.

Layout:
  csrc/      hand-written CUDA kernels + the extern "C" boundary (-> libfaer_b200.so)
  capi.py    ctypes binding of include/faer_b200.h
  linalg.py  host-side mirror of faer::linalg for the hot path (same names / argument meaning)
  solvers.py high-level decompositions (Llt / PartialPivLu / Qr / ColPivQr + the Solve family) over linalg.py
  dist.py    multi-GPU front end: block-column-cyclic layout helpers + distributed LLT

The directory name contains a '-', so import it through the repo-root shim:  `import faer_b200`.
"""
from . import capi, dist, linalg, solvers  # noqa: F401
from .capi import load  # noqa: F401
