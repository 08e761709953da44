"""CPU tier: the sample-format edge's host logic, dsp_b200/csrc/io_plan.h, compiled with g++ alone.

Every shard's copies are replayed with numpy on host byte arrays, as cudaMemcpy2DAsync (or, where io_copy() calls the
rows contiguous, one linear cudaMemcpyAsync) would do them: 1 to 5 shards cut as dspb200_chain_create cuts them (ragged
slabs such as 7 channels over 3), both layouts, both sample types, planar strides equal to and larger than the frames.
The device slab must be what [frames, C] or [C, stride] slicing says, the copy back must land there and nowhere else
(guard-filled padding stays as it was).  Every refusal is refused with its message, f64 interleaved selects no kernel
and no staging, and the page-locked extent covers exactly the rows a call touches.
"""
import ctypes

import numpy as np
import pytest

from accuracy import header_lib

DRIVER = r"""
#include "io_plan.h"
using namespace dspb200;
extern "C" {
int check(int in_fmt, long in_stride, int out_fmt, long out_stride, long frames, long max_out, int same, char *msg, int len)
{
	return io_check(in_fmt, in_stride, out_fmt, out_stride, frames, max_out, same != 0, msg, (size_t) len);
}
// host_off, host_pitch, dev_pitch, width, height, contiguous
void copy(int fmt, long stride, int C, int ch_begin, int ch_count, long frames, long *out)
{
	const IoCopy k = io_copy(fmt, stride, C, ch_begin, ch_count, frames);
	const long v[] = { (long) k.host_off, (long) k.host_pitch, (long) k.dev_pitch, (long) k.width, (long) k.height, k.contiguous ? 1 : 0 };
	for (int i = 0; i < 6; ++i) out[i] = v[i];
}
long stage_bytes(int in_fmt, int out_fmt, int ch_count, long max_frames) { return (long) io_stage_bytes(in_fmt, out_fmt, ch_count, max_frames); }
long host_bytes(int fmt, long stride, int C, long frames) { return (long) io_host_bytes(fmt, stride, C, frames); }
int kernel(int fmt) { return io_kernel(fmt); }
int aligned(unsigned long addr, int fmt) { return io_aligned(addr, fmt) ? 1 : 0; }
}
"""
F64, F32, PLANAR = 0, 1, 0x10
FORMATS = [F64, F32, F64 | PLANAR, F32 | PLANAR]
GUARD = 0xA5


def _name(fmt):
    return ("f32" if fmt & F32 else "f64") + ("_planar" if fmt & PLANAR else "")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = header_lib(tmp_path_factory.mktemp("io_plan"), "ioplan", DRIVER)
    lib.check.argtypes = [ctypes.c_int, ctypes.c_long, ctypes.c_int, ctypes.c_long, ctypes.c_long, ctypes.c_long, ctypes.c_int,
                          ctypes.c_char_p, ctypes.c_int]
    lib.copy.argtypes = [ctypes.c_int, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_long, ctypes.POINTER(ctypes.c_long)]
    lib.stage_bytes.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_long]
    lib.stage_bytes.restype = ctypes.c_long
    lib.host_bytes.argtypes = [ctypes.c_int, ctypes.c_long, ctypes.c_int, ctypes.c_long]
    lib.host_bytes.restype = ctypes.c_long
    lib.kernel.argtypes = [ctypes.c_int]
    lib.aligned.argtypes = [ctypes.c_ulong, ctypes.c_int]
    return lib


def _check(lib, in_fmt, in_stride, out_fmt, out_stride, frames, max_out, same=False):
    msg = ctypes.create_string_buffer(256)
    rc = lib.check(in_fmt, in_stride, out_fmt, out_stride, frames, max_out, int(same), msg, len(msg))
    return rc, msg.value.decode()


def _copy(lib, fmt, stride, C, b, n, frames):
    out = (ctypes.c_long * 6)()
    lib.copy(fmt, stride, C, b, n, frames, out)
    return dict(zip(("host_off", "host_pitch", "dev_pitch", "width", "height", "contiguous"), list(out)))


def _shards(C, n_shards):
    """(ch_begin, ch_count) of each shard, as dspb200_chain_create cuts the channels."""
    n_shards = min(n_shards, C)
    return [(C * i // n_shards, C * (i + 1) // n_shards - C * i // n_shards) for i in range(n_shards)]


def _h2d(host, dev, k):
    """Replay one host -> device copy on byte arrays."""
    if k["contiguous"]:
        n = k["width"] * k["height"]
        dev[:n] = host[k["host_off"]:k["host_off"] + n]
        return
    for r in range(k["height"]):
        h = k["host_off"] + r * k["host_pitch"]
        dev[r * k["dev_pitch"]:r * k["dev_pitch"] + k["width"]] = host[h:h + k["width"]]


def _d2h(dev, host, k):
    if k["contiguous"]:
        n = k["width"] * k["height"]
        host[k["host_off"]:k["host_off"] + n] = dev[:n]
        return
    for r in range(k["height"]):
        h = k["host_off"] + r * k["host_pitch"]
        host[h:h + k["width"]] = dev[r * k["dev_pitch"]:r * k["dev_pitch"] + k["width"]]


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1)


def _host_array(fmt, C, frames, stride, rng):
    """(the caller's whole buffer as its dtype, the [frames, C] view of its samples); planar buffers are [C, stride]
    with the last row cut to its frames, as a caller with an exact allocation may hold it."""
    dt = np.float32 if fmt & F32 else np.float64
    if fmt & PLANAR:
        buf = rng.standard_normal((C - 1) * stride + frames).astype(dt)
        view = np.lib.stride_tricks.as_strided(buf, (C, frames), (stride * buf.itemsize, buf.itemsize))
        return buf, view.T
    buf = rng.standard_normal(frames * C).astype(dt)
    return buf, buf.reshape(frames, C)


CASES = [(C, n, frames, extra) for C, n in ((1, 1), (2, 1), (2, 2), (7, 1), (7, 3), (7, 5), (8, 4), (5, 5), (13, 4))
         for frames in (1, 17) for extra in (0, 3)]


@pytest.mark.parametrize("fmt", FORMATS, ids=_name)
@pytest.mark.parametrize("C,n_shards,frames,extra", CASES, ids=["C%d-s%d-f%d-pad%d" % c for c in CASES])
def test_copy_geometry(lib, fmt, C, n_shards, frames, extra):
    """Each shard's H2D copy brings exactly its channel slab, packed ([frames][n] interleaved, [n][frames] planar), and
    its D2H copy of the same geometry writes exactly that slab back into a guard-filled buffer: after all shards the
    samples are in place and every padding byte (between planar rows and past the last row's frames) is untouched."""
    rng = np.random.default_rng(C * 1000 + n_shards * 100 + frames + extra + fmt)
    stride = (frames + extra) if fmt & PLANAR else 0
    buf, x = _host_array(fmt, C, frames, stride, rng)
    esize = buf.itemsize
    hb = _bytes(buf)
    assert lib.host_bytes(fmt, stride, C, frames) == hb.size
    out = np.full(hb.size, GUARD, dtype=np.uint8)
    for b, n in _shards(C, n_shards):
        k = _copy(lib, fmt, stride, C, b, n, frames)
        assert k["width"] * k["height"] == frames * n * esize, k
        assert k["contiguous"] == (k["host_pitch"] == k["width"]), k
        dev = np.zeros(frames * n * esize, dtype=np.uint8)
        _h2d(hb, dev, k)
        slab = dev.view(buf.dtype)
        want = x[:, b:b + n].T if fmt & PLANAR else x[:, b:b + n]
        assert np.array_equal(slab, np.ascontiguousarray(want).reshape(-1)), (b, n, k)
        _d2h(dev, out, k)
    # everything the samples cover is back, everything else still holds the guard
    covered = np.zeros(hb.size, dtype=bool)
    if fmt & PLANAR:
        elems = np.concatenate([c * stride + np.arange(frames) for c in range(C)])
    else:
        elems = np.arange(buf.size)
    for e in elems:
        covered[e * esize:(e + 1) * esize] = True
    assert np.array_equal(out[covered], hb[covered])
    assert (out[~covered] == GUARD).all()


@pytest.mark.parametrize("fmt", FORMATS, ids=_name)
def test_one_shard_is_one_linear_copy(lib, fmt):
    """A whole-stream slab is contiguous for interleaved buffers and for planar ones whose stride is the frame count, so
    f64 interleaved on one shard keeps the plain call's linear copy; padded planar rows need the 2-D copy."""
    assert _copy(lib, fmt, 100 if fmt & PLANAR else 0, 6, 0, 6, 100)["contiguous"] == 1
    if fmt & PLANAR:
        assert _copy(lib, fmt, 101, 6, 0, 6, 100)["contiguous"] == 0
    else:
        assert _copy(lib, fmt, 0, 6, 0, 3, 100)["contiguous"] == 0


def test_f64_interleaved_keeps_the_plain_path(lib):
    """No edge kernel and no staging for f64 interleaved; every other format converts, and staging is sized by the
    larger side in the caller's element size."""
    assert lib.kernel(F64) == -1
    assert [lib.kernel(f) for f in (F32, F64 | PLANAR, F32 | PLANAR)] == [F32, F64 | PLANAR, F32 | PLANAR]
    assert lib.stage_bytes(F64, F64, 7, 4097) == 0
    assert lib.stage_bytes(F32, F64, 7, 4097) == 7 * 4097 * 4
    assert lib.stage_bytes(F64, F32 | PLANAR, 7, 4097) == 7 * 4097 * 4
    assert lib.stage_bytes(F32, F64 | PLANAR, 7, 4097) == 7 * 4097 * 8
    assert lib.stage_bytes(F64 | PLANAR, F64, 1, 1) == 8


def test_element_alignment(lib):
    """Mode D buffers need the alignment of their element type only."""
    assert lib.aligned(0x1004, F32) and lib.aligned(0x1004, F32 | PLANAR)
    assert not lib.aligned(0x1004, F64) and not lib.aligned(0x1002, F32)
    assert lib.aligned(0x1008, F64 | PLANAR)


@pytest.mark.parametrize("in_fmt", FORMATS, ids=_name)
@pytest.mark.parametrize("out_fmt", FORMATS, ids=_name)
def test_accepted(lib, in_fmt, out_fmt):
    """All 16 pairs with exact and padded strides, and in place with the same format and stride."""
    for pad in (0, 5):
        si = 100 + pad if in_fmt & PLANAR else 0
        so = 120 + pad if out_fmt & PLANAR else 0
        assert _check(lib, in_fmt, si, out_fmt, so, 100, 120) == (0, "")
    if in_fmt == out_fmt:
        s = 130 if in_fmt & PLANAR else 0
        assert _check(lib, in_fmt, s, out_fmt, s, 100, 120, same=True) == (0, "")


REFUSALS = {
    "unknown_in_bits": ((0x2, 0, F64, 0, 10, 10, False), "unknown format bits"),
    "unknown_out_bits": ((F64, 0, 0x100, 0, 10, 10, False), "unknown format bits"),
    "f16_like_bits": ((0x3, 0, F32, 0, 10, 10, False), "unknown format bits"),
    "interleaved_in_stride": ((F32, 10, F32, 0, 10, 10, False), "interleaved input takes stride 0"),
    "interleaved_out_stride": ((F32, 0, F64, 12, 10, 10, False), "interleaved output takes stride 0"),
    "short_in_stride": ((F32 | PLANAR, 9, F32, 0, 10, 10, False), "planar input stride 9 is shorter than the 10 frames"),
    "short_out_stride": ((F32, 0, F32 | PLANAR, 10, 10, 11, False), "planar output stride 10 is shorter than the chain's max_out_frames 11"),
    "in_place_across_types": ((F32, 0, F64, 0, 10, 10, True), "in place needs the same format and stride"),
    "in_place_across_layouts": ((F64 | PLANAR, 10, F64, 0, 10, 10, True), "in place needs the same format and stride"),
    "in_place_across_strides": ((F32 | PLANAR, 10, F32 | PLANAR, 12, 10, 10, True), "in place needs the same format and stride"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refused(lib, case):
    args, message = REFUSALS[case]
    rc, msg = _check(lib, *args)
    assert rc == -1 and message in msg, (case, msg)


def test_edge_kernels_sass(tmp_path):
    """edge.cu compiled for sm_90a as the library compiles it: the conversions are F2F.F32.F64 (round to nearest, no
    .FTZ) and F2F.F64.F32, and no edge kernel spills."""
    import os
    import shutil
    import subprocess
    from accuracy import CSRC
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(nvcc) or not os.path.exists(cuobjdump):
        pytest.skip("no CUDA toolkit")
    obj = tmp_path / "edge.o"
    r = subprocess.run([nvcc, "-c", "-Xcompiler", "-fPIC", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-Xptxas", "-v", os.path.join(CSRC, "edge.cu"), "-o", str(obj)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, check=True)
    props = [line for line in r.stdout.splitlines() if "spill stores" in line]
    assert len(props) == 6 and all("0 bytes spill stores, 0 bytes spill loads" in line for line in props), r.stdout
    sass = subprocess.run([cuobjdump, "-sass", str(obj)], stdout=subprocess.PIPE, text=True, check=True).stdout
    f2f = [line.split("F2F", 1)[1].split()[0] for line in sass.splitlines() if "F2F" in line]
    assert ".F32.F64" in f2f and ".F64.F32" in f2f, sorted(set(f2f))
    assert not any("FTZ" in k for k in f2f), sorted(set(f2f))
