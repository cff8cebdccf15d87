"""btle_b200 — CUDA-native (H100, sm_90a) BLE receive baseband (drop-in for the btle_rx receive chain)."""
from ._native import BtleError, CAND_DTYPE, CFG_DTYPE, CODED_CAND_DTYPE, CODED_REC_DTYPE, DIR_DTYPE, REC_DTYPE  # noqa: F401
from .rx import BtleRx, make_cfgs  # noqa: F401

__all__ = ["BtleRx", "BtleError", "make_cfgs", "REC_DTYPE", "CFG_DTYPE", "DIR_DTYPE", "CAND_DTYPE", "CODED_CAND_DTYPE", "CODED_REC_DTYPE"]
