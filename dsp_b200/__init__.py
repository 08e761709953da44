"""dsp_b200 -- H100 (sm_90a) implementation of bmc0/dsp's per-block effects-chain hot path.

The product is libdspb200.so (hand-written CUDA behind the C ABI of include/dsp_b200.h) plus the
C shim under shim/ that exposes it through the reference's own `struct effect` surface.  This
Python package is the thin binding used by tests and bench.py; it has no CPU path.
"""
from .lib import (Chain, DspB200Error, debug_serialize, debug_stall, PinnedArray, biquad_design, device_count, hilbert_taps,  # noqa: F401
                  kernel_launches, last_error, lib, profile_enable, profile_read, resample_params, copy_counts,
                  STALL_HOT, STALL_MAIN, STALL_SIDE, STALL_SIDE2, IO_F32, IO_F64, IO_PLANAR, io_format)
