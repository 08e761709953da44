"""ctypes binding of libdspb200.so (include/dsp_b200.h).

There is no CPU path: if the CUDA library is missing or no device is usable, constructing a
Chain raises.  numpy arrays are host buffers (mode A); raw device pointers + a cudaStream_t
(e.g. from torch tensors / torch.cuda.current_stream().cuda_stream) are mode D.  Chain.run_io and Chain.run_tensor
take float32 or float64 blocks, interleaved [frames, channels] or planar [channels, frames] (the _io calls).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DSP_B200_LIB") or os.path.join(_HERE, "libdspb200.so")   # DSP_B200_LIB: a measurement variant (build.build_variant)

_lib = None

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)
_lp = C.POINTER(C.c_long)

# name -> (restype, argtypes); must list every function include/dsp_b200.h declares
SIGNATURES = {
    "dspb200_version": (C.c_char_p, []),
    "dspb200_last_error": (C.c_char_p, []),
    "dspb200_device_count": (C.c_int, []),
    "dspb200_host_alloc": (C.c_void_p, [C.c_size_t]),
    "dspb200_host_alloc_wc": (C.c_void_p, [C.c_size_t]),
    "dspb200_host_free": (None, [C.c_void_p]),
    "dspb200_kernel_launches": (C.c_longlong, []),
    "dspb200_profile_enable": (None, [C.c_int]),
    "dspb200_debug_serialize": (None, [C.c_int]),
    "dspb200_debug_stall": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int]),
    "dspb200_profile_read": (C.c_int, [C.c_char_p, C.POINTER(C.c_double), _lp]),
    "dspb200_chain_create": (C.c_void_p, [C.c_int, C.c_int, _ip, C.c_int, C.c_int]),
    "dspb200_chain_destroy": (None, [C.c_void_p]),
    "dspb200_chain_absorb": (C.c_int, [C.c_void_p, C.c_void_p]),
    "dspb200_chain_n_ops": (C.c_int, [C.c_void_p]),
    "dspb200_chain_describe": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "dspb200_chain_n_shards": (C.c_int, [C.c_void_p]),
    "dspb200_chain_shard_info": (C.c_int, [C.c_void_p, C.c_int, _ip, _ip, _ip]),
    "dspb200_chain_out_fs": (C.c_int, [C.c_void_p]),
    "dspb200_chain_add_gain": (C.c_int, [C.c_void_p, _dp, _dp]),
    "dspb200_chain_add_biquad": (C.c_int, [C.c_void_p, C.c_int, _dp]),
    "dspb200_chain_add_fir": (C.c_int, [C.c_void_p, C.c_char_p, _dp, C.c_int, C.c_long, C.c_long, C.c_long]),
    "dspb200_chain_add_align": (C.c_int, [C.c_void_p, _lp, C.c_long]),
    "dspb200_chain_inplace_ok": (C.c_int, [C.c_void_p]),
    "dspb200_copy_counts": (None, [C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
    "dspb200_chain_add_resample": (C.c_int, [C.c_void_p, C.c_int, C.c_double]),
    "dspb200_chain_max_out_frames": (C.c_long, [C.c_void_p, C.c_long]),
    "dspb200_chain_run_host": (C.c_long, [C.c_void_p, C.c_long, C.c_void_p, C.c_void_p]),
    "dspb200_chain_run_device": (C.c_long, [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dspb200_chain_join": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    "dspb200_debug_read": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_longlong), C.c_int]),
    "dspb200_chain_drain_host": (C.c_long, [C.c_void_p, C.c_long, C.c_void_p]),
    "dspb200_chain_reset": (None, [C.c_void_p]),
    "dspb200_chain_sync": (C.c_int, [C.c_void_p]),
    "dspb200_chain_submit_host": (C.c_long, [C.c_void_p, C.c_long, C.c_void_p, C.c_void_p, C.POINTER(C.c_ulonglong)]),
    "dspb200_chain_wait": (C.c_int, [C.c_void_p, C.c_ulonglong]),
    "dspb200_chain_run_host_io": (C.c_long, [C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int, C.c_long]),
    "dspb200_chain_submit_host_io": (C.c_long, [C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int, C.c_long,
                                                C.POINTER(C.c_ulonglong)]),
    "dspb200_chain_run_device_io": (C.c_long, [C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int, C.c_long, C.c_void_p, C.c_int,
                                               C.c_long, C.c_void_p]),
    "dspb200_chain_drain_host_io": (C.c_long, [C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_long]),
    "dspb200_biquad_design": (C.c_int, [C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int, _dp]),
    "dspb200_hilbert_taps": (C.c_int, [C.c_long, C.c_double, _dp]),
    "dspb200_resample_params": (C.c_int, [C.c_int, C.c_int, C.c_double, _lp]),
    "dspb200_test_rfft": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dspb200_test_irfft": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
}


class DspB200Error(RuntimeError):
    pass


# sample formats of the _io calls (DSPB200_IO_* in include/dsp_b200.h): a type | a layout
IO_F64, IO_F32, IO_PLANAR = 0, 1, 0x10


def io_format(dtype, planar):
    """The DSPB200_IO_* format of samples of `dtype` (float32 or float64) in the given layout."""
    dtype = np.dtype(dtype)
    if dtype not in (np.float32, np.float64):
        raise DspB200Error("sample formats are float32 and float64, not %s" % dtype)
    return (IO_F32 if dtype == np.float32 else IO_F64) | (IO_PLANAR if planar else 0)


def _io_stride(shape, strides, itemsize, planar):
    """(rows stride in elements for the ABI, True when the array's layout needs no copy) of a 2-D array."""
    if planar:
        ok = shape[1] <= 1 or strides[1] == itemsize
        ok = ok and strides[0] % itemsize == 0 and strides[0] >= 0 and (shape[0] <= 1 or strides[0] // itemsize >= shape[1])
        return (strides[0] // itemsize if shape[0] > 1 else shape[1]), ok
    ok = (shape[1] <= 1 or strides[1] == itemsize) and (shape[0] <= 1 or strides[0] == shape[1] * itemsize)
    return 0, ok


def lib():
    """Load libdspb200.so; raises (never falls back) when it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise DspB200Error("libdspb200.so not built: run `python -m dsp_b200.build` (needs nvcc)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def last_error():
    return lib().dspb200_last_error().decode(errors="replace")


def device_count():
    return lib().dspb200_device_count()


def kernel_launches():
    return lib().dspb200_kernel_launches()


def profile_enable(on):
    lib().dspb200_profile_enable(1 if on else 0)


def debug_serialize(on):
    lib().dspb200_debug_serialize(1 if on else 0)


# roles of debug_stall (DSPB200_STALL_* in include/dsp_b200.h)
STALL_MAIN, STALL_SIDE, STALL_SIDE2, STALL_HOT = 1, 2, 4, 8


def debug_stall(roles, microseconds=0, period=1, phase=0):
    """Test aid: FIR operators delay the streams in `roles` by `microseconds` before their first FIR launch of every
    level-0 block blk % period == phase (roles = 0: off).  Results must not change."""
    _check(lib().dspb200_debug_stall(int(roles), int(microseconds), int(period), int(phase)), "debug_stall")


def profile_read(name):
    """-> (total milliseconds, launches) of the named kernel since the last read."""
    ms, n = C.c_double(), C.c_long()
    lib().dspb200_profile_read(name.encode(), C.byref(ms), C.byref(n))
    return ms.value, n.value


def _check(rc, what):
    if rc is None or (isinstance(rc, int) and rc < 0):
        raise DspB200Error("%s failed: %s" % (what, last_error()))
    return rc


def _as_dp(a):
    return a.ctypes.data_as(_dp)


class PinnedArray:
    """float64 numpy view over page-locked host memory from dspb200_host_alloc()."""

    def __init__(self, shape, write_combined=False):
        self.shape = tuple(int(s) for s in shape)
        n = int(np.prod(self.shape)) if self.shape else 1
        alloc = lib().dspb200_host_alloc_wc if write_combined else lib().dspb200_host_alloc
        self.ptr = alloc(max(n, 1) * 8)
        if not self.ptr:
            raise DspB200Error("host_alloc failed: " + last_error())
        buf = (C.c_double * max(n, 1)).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=np.float64, count=n).reshape(self.shape)

    def free(self):
        if self.ptr:
            self.array = None
            lib().dspb200_host_free(self.ptr)
            self.ptr = None


class Chain:
    """Device-side twin of a run of consecutive GPU effects of a reference effects_chain."""

    def __init__(self, fs, channels, devices=None, slabs_per_device=1):
        L = lib()
        devs = list(devices) if devices else []
        arr = (C.c_int * len(devs))(*devs) if devs else None
        self.h = L.dspb200_chain_create(int(fs), int(channels), arr, len(devs), int(slabs_per_device))
        if not self.h:
            raise DspB200Error("chain_create failed: " + last_error())
        self.fs = int(fs)
        self.channels = int(channels)

    # -- construction -------------------------------------------------------------------
    def add_gain(self, mult, add=None):
        mult = np.ascontiguousarray(np.broadcast_to(np.asarray(mult, dtype=np.float64), (self.channels,)))
        addp = None
        if add is not None:
            add = np.ascontiguousarray(np.broadcast_to(np.asarray(add, dtype=np.float64), (self.channels,)))
            addp = _as_dp(add)
        _check(lib().dspb200_chain_add_gain(self.h, _as_dp(mult), addp), "add_gain")
        return self

    def add_biquad(self, coefs):
        """coefs: [stages, channels, 5] (or [stages, 5], same section on every channel)."""
        coefs = np.asarray(coefs, dtype=np.float64)
        if coefs.ndim == 2:
            coefs = np.repeat(coefs[:, None, :], self.channels, axis=1)
        assert coefs.shape[1:] == (self.channels, 5), coefs.shape
        coefs = np.ascontiguousarray(coefs)
        _check(lib().dspb200_chain_add_biquad(self.h, coefs.shape[0], _as_dp(coefs)), "add_biquad")
        return self

    def add_fir(self, taps, selector=None, latency=0, block_hint=0):
        """taps: [frames] or [frames, filter_channels]; selector: per-channel truthy mask or None."""
        taps = np.asarray(taps, dtype=np.float64)
        if taps.ndim == 1:
            taps = taps[:, None]
        taps = np.ascontiguousarray(taps)
        sel = None
        if selector is not None:
            sel = bytes(bytearray(1 if s else 0 for s in selector))
            assert len(sel) == self.channels
        _check(lib().dspb200_chain_add_fir(self.h, sel, _as_dp(taps), taps.shape[1], taps.shape[0], int(latency), int(block_hint)), "add_fir")
        return self

    def add_align(self, delay, discard_frames=0):
        """delay: per-channel whole-frame delays (align.c / delay.c); discard_frames dropped at the head of the stream."""
        d = (C.c_long * self.channels)(*[int(v) for v in np.broadcast_to(np.asarray(delay), (self.channels,))])
        _check(lib().dspb200_chain_add_align(self.h, d, int(discard_frames)), "add_align")
        return self

    def add_resample(self, out_fs, bandwidth=0.0):
        _check(lib().dspb200_chain_add_resample(self.h, int(out_fs), float(bandwidth)), "add_resample")
        return self

    def absorb(self, other):
        _check(lib().dspb200_chain_absorb(self.h, other.h), "absorb")
        return self

    # -- introspection ------------------------------------------------------------------
    @property
    def n_ops(self):
        return lib().dspb200_chain_n_ops(self.h)

    def describe(self):
        """Operators of shard 0 with their plans (list of dicts)."""
        import json
        buf = C.create_string_buffer(1 << 16)
        lib().dspb200_chain_describe(self.h, buf, len(buf))
        return json.loads(buf.value.decode())

    @property
    def n_shards(self):
        return lib().dspb200_chain_n_shards(self.h)

    @property
    def out_fs(self):
        return lib().dspb200_chain_out_fs(self.h)

    def shard_info(self, shard):
        d, b, n = C.c_int(), C.c_int(), C.c_int()
        _check(lib().dspb200_chain_shard_info(self.h, shard, C.byref(d), C.byref(b), C.byref(n)), "shard_info")
        return d.value, b.value, n.value

    def max_out_frames(self, frames):
        return lib().dspb200_chain_max_out_frames(self.h, int(frames))

    # -- running ------------------------------------------------------------------------
    def run(self, x, out=None):
        """Mode A: x [frames, channels] float64 host array -> [out_frames, channels]."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        frames = x.shape[0]
        if out is None:
            out = np.empty((max(self.max_out_frames(frames), frames, 1), self.channels), dtype=np.float64)
        n = _check(lib().dspb200_chain_run_host(self.h, frames, x.ctypes.data, out.ctypes.data), "run_host")
        return out[:n]

    def run_raw(self, frames, in_ptr, out_ptr):
        return _check(lib().dspb200_chain_run_host(self.h, int(frames), in_ptr, out_ptr), "run_host")

    def submit_raw(self, frames, in_ptr, out_ptr):
        """run_raw without the wait: returns (out_frames, ticket); buffers stay busy until wait(ticket)."""
        t = C.c_ulonglong(0)
        n = _check(lib().dspb200_chain_submit_host(self.h, int(frames), in_ptr, out_ptr, C.byref(t)), "submit_host")
        return n, t.value

    def wait(self, ticket):
        _check(lib().dspb200_chain_wait(self.h, int(ticket)), "wait")

    def run_io(self, x, planar=False, out=None):
        """Mode A in the caller's format: x a float32 or float64 host array, [frames, channels] or, planar,
        [channels, frames] (rows may be further apart than `frames`).  Returns `out` (or a new array of x's dtype) cut to
        the returned frames, in the same layout.  out may be wider than the result; its dtype sets the output format."""
        x = np.asarray(x)
        if x.ndim != 2 or x.shape[0 if planar else 1] != self.channels:
            raise DspB200Error("run_io: expected %s, got shape %s" % ("[channels, frames]" if planar else "[frames, channels]", x.shape))
        in_fmt = io_format(x.dtype, planar)
        in_stride, ok = _io_stride(x.shape, x.strides, x.itemsize, planar)
        if not ok:
            x = np.ascontiguousarray(x)
            in_stride, _ = _io_stride(x.shape, x.strides, x.itemsize, planar)
        frames = x.shape[1 if planar else 0]
        n_out = max(self.max_out_frames(frames), frames if not planar else 0, 1)
        if out is None:
            out = np.empty((self.channels, n_out) if planar else (n_out, self.channels), dtype=x.dtype)
        out_fmt = io_format(out.dtype, planar)
        out_stride, ok = _io_stride(out.shape, out.strides, out.itemsize, planar)
        if not ok or out.shape[0 if planar else 1] != self.channels:
            raise DspB200Error("run_io: out must be a writable %s array with unit-stride rows" % ("[channels, W]" if planar else "[frames, channels]"))
        n = _check(lib().dspb200_chain_run_host_io(self.h, frames, x.ctypes.data, in_fmt, in_stride, out.ctypes.data, out_fmt, out_stride),
                   "run_host_io")
        return out[:, :n] if planar else out[:n]

    def run_io_raw(self, frames, in_ptr, in_fmt, in_stride, out_ptr, out_fmt, out_stride):
        """run_raw in the caller's formats (IO_* | IO_PLANAR); strides in elements, 0 for interleaved buffers."""
        return _check(lib().dspb200_chain_run_host_io(self.h, int(frames), in_ptr, int(in_fmt), int(in_stride), out_ptr, int(out_fmt),
                                                      int(out_stride)), "run_host_io")

    def submit_io_raw(self, frames, in_ptr, in_fmt, in_stride, out_ptr, out_fmt, out_stride):
        """submit_raw in the caller's formats: returns (out_frames, ticket); buffers stay busy until wait(ticket)."""
        t = C.c_ulonglong(0)
        n = _check(lib().dspb200_chain_submit_host_io(self.h, int(frames), in_ptr, int(in_fmt), int(in_stride), out_ptr, int(out_fmt),
                                                      int(out_stride), C.byref(t)), "submit_host_io")
        return n, t.value

    def run_device_io(self, shard, frames, d_in, in_fmt, in_stride, d_out, out_fmt, out_stride, stream=None):
        """run_device in the caller's formats (raw device pointers, strides in elements)."""
        return _check(lib().dspb200_chain_run_device_io(self.h, int(shard), int(frames), d_in, int(in_fmt), int(in_stride), d_out,
                                                        int(out_fmt), int(out_stride), stream), "run_device_io")

    def run_tensor(self, x, planar=True, out=None):
        """Mode D on torch.cuda.current_stream(): x a CUDA tensor, float32 or float64, [channels, T] (planar, the
        default) or [T, channels].  Returns `out` (or a new tensor of x's dtype) cut to the returned frames, in the same
        layout; out may be wider than the result and in place (out is x) where the chain allows it.  Single-shard
        chains only."""
        import torch
        if self.n_shards != 1:
            raise DspB200Error("run_tensor: the chain has %d shards; run_tensor drives single-shard chains (use run_device_io per shard)"
                               % self.n_shards)
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dim() == 2):
            raise DspB200Error("run_tensor: expected a 2-D CUDA tensor")
        if x.shape[0 if planar else 1] != self.channels:
            raise DspB200Error("run_tensor: expected %s with %d channels, got %s" % ("[channels, T]" if planar else "[T, channels]",
                                                                                    self.channels, tuple(x.shape)))
        dev = self.shard_info(0)[0]
        if x.device.index != dev:
            raise DspB200Error("run_tensor: the chain runs on cuda:%d, x is on %s" % (dev, x.device))
        isz = x.element_size()
        in_fmt = io_format(str(x.dtype).replace("torch.", ""), planar)
        in_stride, ok = _io_stride(tuple(x.shape), tuple(s * isz for s in x.stride()), isz, planar)
        if not ok:
            x = x.contiguous()
            in_stride, _ = _io_stride(tuple(x.shape), tuple(s * isz for s in x.stride()), isz, planar)
        frames = x.shape[1 if planar else 0]
        n_out = max(self.max_out_frames(frames), 1)
        if out is None:
            out = torch.empty((self.channels, n_out) if planar else (n_out, self.channels), dtype=x.dtype, device=x.device)
        osz = out.element_size()
        out_fmt = io_format(str(out.dtype).replace("torch.", ""), planar)
        out_stride, ok = _io_stride(tuple(out.shape), tuple(s * osz for s in out.stride()), osz, planar)
        if not ok or out.device != x.device or out.shape[0 if planar else 1] != self.channels:
            raise DspB200Error("run_tensor: out must be a %s tensor on %s with unit-stride rows" % ("[channels, W]" if planar else "[T, channels]",
                                                                                                  x.device))
        with torch.cuda.device(x.device):
            stream = torch.cuda.current_stream().cuda_stream
        n = self.run_device_io(0, frames, x.data_ptr(), in_fmt, in_stride, out.data_ptr(), out_fmt, out_stride, stream)
        return out[:, :n] if planar else out[:n]

    def run_device(self, shard, frames, d_in, d_out, stream=None):
        """Mode D: raw device pointers (ints), asynchronous on `stream` (cudaStream_t as int)."""
        return _check(lib().dspb200_chain_run_device(self.h, int(shard), int(frames), d_in, d_out, stream), "run_device")

    def join(self, shard, stream=None):
        """Make `stream` wait for everything the shard's operators have enqueued on streams of their own."""
        _check(lib().dspb200_chain_join(self.h, int(shard), stream), "join")

    def debug_read(self, shard=0, op_index=0, max_values=8 * 1024):
        """Operator-specific device counters (measurement hook); numpy int64 array."""
        buf = (C.c_longlong * max_values)()
        n = lib().dspb200_debug_read(self.h, int(shard), int(op_index), buf, max_values)
        return np.array(buf[:max(n, 0)], dtype=np.int64)

    def drain(self, frames):
        """One drain2 poll (resample.c:163-188); None when dry."""
        out = np.empty((max(self.max_out_frames(frames), 1), self.channels), dtype=np.float64)
        n = lib().dspb200_chain_drain_host(self.h, int(frames), out.ctypes.data)
        if n == -1:
            return None
        if n < 0:
            raise DspB200Error("drain_host failed: " + last_error())
        return out[:n].copy()

    def drain_io(self, frames, dtype=np.float64, planar=False):
        """drain() in the caller's format: a [frames, channels] or, planar, [channels, frames] array of `dtype`; None when
        dry."""
        n_out = max(self.max_out_frames(frames), 1)
        out = np.empty((self.channels, n_out) if planar else (n_out, self.channels), dtype=dtype)
        fmt = io_format(dtype, planar)
        n = lib().dspb200_chain_drain_host_io(self.h, int(frames), out.ctypes.data, fmt, n_out if planar else 0)
        if n == -1:
            return None
        if n < 0:
            raise DspB200Error("drain_host_io failed: " + last_error())
        return (out[:, :n] if planar else out[:n]).copy()

    def process(self, x, block, drain_frames=0):
        """Whole stream in `block`-frame calls, then `drain_frames` of silence (the chain's
        drain_samples total, effects_chain.c:1193-1198), then drain2 polling.  Returns
        (concatenated output, per-call frame counts)."""
        outs, counts = [], []
        for i in range(0, x.shape[0], block):
            y = self.run(x[i:i + block]).copy()
            outs.append(y)
            counts.append(y.shape[0])
        left = drain_frames
        while left > 0:
            f = min(block, left)
            left -= f
            y = self.run(np.zeros((f, self.channels))).copy()
            outs.append(y)
            counts.append(y.shape[0])
        while True:
            y = self.drain(block)
            if y is None:
                break
            outs.append(y)
            counts.append(y.shape[0])
        y = np.concatenate(outs, axis=0) if outs else np.zeros((0, self.channels))
        return y, counts

    def reset(self):
        lib().dspb200_chain_reset(self.h)

    def sync(self):
        _check(lib().dspb200_chain_sync(self.h), "sync")

    def close(self):
        if getattr(self, "h", None):
            lib().dspb200_chain_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def copy_counts():
    """(host->device, device->host) block copies issued so far by this process."""
    a, b = C.c_longlong(), C.c_longlong()
    lib().dspb200_copy_counts(C.byref(a), C.byref(b))
    return a.value, b.value


def biquad_design(type_, fs, arg0, arg1=0.0, arg2=0.0, arg3=0.0, width_type=1):
    c = np.zeros(5)
    _check(lib().dspb200_biquad_design(int(type_), float(fs), float(arg0), float(arg1), float(arg2), float(arg3), int(width_type), _as_dp(c)), "biquad_design")
    return c


def hilbert_taps(taps, angle=-np.pi / 2):
    h = np.zeros(int(taps))
    _check(lib().dspb200_hilbert_taps(int(taps), float(angle), _as_dp(h)), "hilbert_taps")
    return h


def resample_params(fs_in, fs_out, bandwidth=0.0):
    out = (C.c_long * 8)()
    _check(lib().dspb200_resample_params(int(fs_in), int(fs_out), float(bandwidth), out), "resample_params")
    keys = ("n", "d", "m", "in_len", "out_len", "sinc_len", "out_delay", "taps_per_phase")
    return dict(zip(keys, [int(v) for v in out]))
