"""polypolish_b200 — H100-native (Hopper, sm_90a) implementation of Polypolish's alignment-pileup-and-vote path.

The product is the C-ABI shared library build/libpolypolish_b200.so (include/pp_abi.h) and the `polypolish`
CLI built next to it.  This package is only the thin ctypes mirror of that ABI used by the tests and bench.py;
it contains no compute and no fallback: importing works anywhere, but every compute call raises unless the
CUDA library is built and an H100 (compute capability 9.0) is visible.
"""
from .api import (Context, PolypolishError, batch, filter_sams, lib, lib_path, load_fasta, pack_sams, polish,  # noqa: F401
                  polish_files)

__version__ = "0.6.1-b200"
