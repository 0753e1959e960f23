"""bevbert_b200 -- H100-native implementation of BEVBert's hybrid-map cross-modal encoder hot path.

Layout:
  csrc/ + libbevbert_b200.so   hand-written sm_90a kernels behind the C ABI (include/bevbert_b200.h)
  _lib.py                      ctypes loader (fails loudly when the library is missing)
  kernels.py                   one thin tensor-level wrapper per C-ABI entry point
  blocks.py                    forward/backward of the encoder blocks, composed from kernels
  model/                       the reference's class surface (vilmodel / pretrain_cmt / bev_utils / ops)
  synth.py                     synthetic batches in the reference's collate layout
  config.py                    model configuration (the keys the path reads)
"""
from .config import make_config  # noqa: F401

__version__ = "0.1.0"
