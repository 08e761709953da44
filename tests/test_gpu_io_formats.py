"""GPU tier: the sample-format edge (the _io calls, edge.cu) in every pair of formats.

The contract is out_io == fmt_out(run(f64_interleaved(x))): a chain called through an _io entry point with x in the
input format must give, bit for bit (NaN by isnan), what an identically built chain gives through today's f64
interleaved calls with the same call sizes, converted to the output format by numpy (astype: round to nearest even,
overflow to +-Inf).  float32 -> float64 is exact and no kernel here uses atomics, so any difference is a bug.

Chains (7 channels, or 8 for the reduced headline): gain/add, a 10-stage biquad cascade, a short direct-form FIR, a
fir_p of one level and one of several, hilbert, resample up and down, align with a discard, biquad x8 -> fir_p ->
resample, and 131072-tap fir_p.  Calls: ragged sizes from 1 frame up, a reset() mid-stream and the drain through
drain_host_io.  Modes: the synchronous host call (1 and 3 slabs), submit/wait with 12 tickets outstanding over the
ring of 8, and Mode D on a non-default stream with a torch.cuda._sleep before each call, on 4-byte-aligned f32 rows.
Every host buffer and Mode D buffer is guard-filled: padding between planar rows and rows past the returned frames
must keep the guard, d_in its input.  Counts: one H2D and one D2H per shard and call, and the launches of the plain
calls plus one edge kernel per converted side and shard; f64 interleaved adds nothing.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F64, F32, PLANAR = 0, 1, 0x10
FORMATS = [F64, F32, F64 | PLANAR, F32 | PLANAR]
PAIRS = [(a, b) for a in FORMATS for b in FORMATS]
CANARY = {np.float64: 0x7FF80000DEADBEEF, np.float32: 0x7FC0BEEF}   # quiet NaNs no kernel computes
UINT = {np.float64: np.uint64, np.float32: np.uint32}
SLEEP_CYCLES = 200000
PAD = 3             # planar stride = frames + PAD; interleaved outputs get PAD guard rows
SIZES = [1, 700, 4096, 33, 4097, 5, 2048, 1000]
RESET_AT = 4        # reset() before this call


def _name(fmt):
    return ("f32" if fmt & F32 else "f64") + ("p" if fmt & PLANAR else "i")


def _dtype(fmt):
    return np.float32 if fmt & F32 else np.float64


def _cast(y, fmt):
    """numpy's conversion of f64 samples to the format's type."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(y, dtype=np.float64).astype(_dtype(fmt))


def _same(got, want, what):
    """Bit for bit, NaN by isnan."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), (what, "NaN positions differ")
    u = UINT[want.dtype.type]
    bad = (got.view(u) != want.view(u)) & ~wn
    assert not bad.any(), (what, "first difference at", np.argwhere(bad)[:3], got[bad][:3], want[bad][:3])


# ------------------------------------------------------------------------------------------------------------
# chains
# ------------------------------------------------------------------------------------------------------------
def _taps(n, C, seed):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, C)) * np.exp(-np.arange(n) / (n / 4.0))[:, None] * 0.1


def _sections(gpu_lib, fs, n):
    return np.array([gpu_lib.biquad_design(13, fs, 60.0 * 1.7 ** k, 0.8 + 0.1 * k, (-1) ** k * 3.0) for k in range(n)])


def _build(gpu_lib, name, slabs, devices=None):
    C = 8 if name == "headline" else 7
    fs = 48000 if name == "resample_down" else 44100
    ch = gpu_lib.Chain(fs, C, devices=devices, slabs_per_device=slabs)
    if name == "gain":
        ch.add_gain(0.5 + np.arange(C) / 8.0, (np.arange(C) - 3) / 16.0)
    elif name == "biquad10":
        ch.add_biquad(_sections(gpu_lib, fs, 10))
    elif name == "fir_direct":
        ch.add_fir(_taps(32, C, 1))
    elif name == "fir_p_short":
        ch.add_fir(_taps(3000, C, 2), block_hint=4096)
    elif name == "fir_p_multi":
        ch.add_fir(_taps(20000, C, 3), block_hint=64)
    elif name == "hilbert":
        ch.add_fir(gpu_lib.hilbert_taps(1001))
    elif name == "resample_up":
        ch.add_resample(48000)
    elif name == "resample_down":
        ch.add_resample(44100)
    elif name == "align":
        ch.add_align([0, 1, 700, 5000, 3, 0, 2], 1000)
    elif name == "combo":
        ch.add_biquad(_sections(gpu_lib, fs, 8)).add_fir(_taps(65536, C, 4), block_hint=4096).add_resample(48000)
    elif name == "headline":
        ch.add_fir(_taps(131072, C, 5), block_hint=4096)
    return ch


CHAINS = ["gain", "biquad10", "fir_direct", "fir_p_short", "fir_p_multi", "hilbert", "resample_up", "resample_down", "align",
          "combo", "headline"]


def _input(name, C, fmt_type):
    """The stream [N, C] as the caller holds it (float32 or float64), with every value exact in float32."""
    rng = np.random.default_rng(len(name) * 31 + C)
    x = (rng.standard_normal((sum(SIZES), C)) * 0.25).astype(np.float32)
    return x.astype(fmt_type)


# ------------------------------------------------------------------------------------------------------------
# caller buffers in a format, guard-filled
# ------------------------------------------------------------------------------------------------------------
class Buf:
    """A host buffer of C channels and `frames` frames in `fmt`: planar [C, frames + PAD], interleaved
    [frames + PAD, C]; everything starts as the canary."""

    def __init__(self, fmt, C, frames):
        self.fmt, self.C, self.frames = fmt, C, frames
        dt = _dtype(fmt)
        self.stride = frames + PAD if fmt & PLANAR else 0
        self.arr = np.empty((C, self.stride) if fmt & PLANAR else (frames + PAD, C), dtype=dt)
        self.arr.view(UINT[dt]).fill(CANARY[dt])

    def put(self, x):
        """x [frames, C] into the buffer."""
        if self.fmt & PLANAR:
            self.arr[:, :x.shape[0]] = x.T
        else:
            self.arr[:x.shape[0]] = x

    def get(self, n):
        return (self.arr[:, :n].T if self.fmt & PLANAR else self.arr[:n]).copy()

    def guards_kept(self, n):
        u = self.arr.view(UINT[self.arr.dtype.type])
        rest = u[:, n:] if self.fmt & PLANAR else u[n:]
        return bool((rest == CANARY[self.arr.dtype.type]).all())

    @property
    def ptr(self):
        return self.arr.ctypes.data


def _counts(gpu_lib):
    return gpu_lib.copy_counts() + (gpu_lib.kernel_launches(),)


def _delta(a, b):
    return tuple(y - x for x, y in zip(a, b))


def _run_host(gpu_lib, ch, x, in_fmt, out_fmt, old_api, drain_block=1024):
    """The calls of SIZES (reset before RESET_AT), then drain polls: (outputs per call, (h2d, d2h, launches) per call).
    old_api: today's run_raw / drain on f64 interleaved buffers (in_fmt and out_fmt must be F64)."""
    outs, counts, pos = [], [], 0
    for i, f in enumerate(SIZES):
        if i == RESET_AT:
            ch.reset()
        bi, bo = Buf(in_fmt, ch.channels, f), Buf(out_fmt, ch.channels, max(ch.max_out_frames(f), f, 1))
        bi.put(x[pos:pos + f])
        before_in = bi.arr.copy()
        c0 = _counts(gpu_lib)
        if old_api:
            n = ch.run_raw(f, bi.ptr, bo.ptr)
        else:
            n = ch.run_io_raw(f, bi.ptr, in_fmt, bi.stride, bo.ptr, out_fmt, bo.stride)
        counts.append(_delta(c0, _counts(gpu_lib)))
        assert bo.guards_kept(n), ("call %d wrote past its %d frames" % (i, n), _name(in_fmt), _name(out_fmt))
        assert np.array_equal(before_in.view(np.uint8), bi.arr.view(np.uint8)), ("call %d changed its input" % i)
        outs.append(bo.get(n))
        pos += f
    while True:
        bo = Buf(out_fmt, ch.channels, max(ch.max_out_frames(drain_block), 1))
        c0 = _counts(gpu_lib)
        fn = gpu_lib.lib().dspb200_chain_drain_host_io
        n = fn(ch.h, drain_block, bo.ptr, out_fmt, bo.stride) if not old_api else gpu_lib.lib().dspb200_chain_drain_host(ch.h, drain_block, bo.ptr)
        assert n >= -1, gpu_lib.last_error()
        if n == -1:
            break
        counts.append(_delta(c0, _counts(gpu_lib)))
        assert bo.guards_kept(n), ("drain wrote past its %d frames" % n, _name(out_fmt))
        outs.append(bo.get(n))
    return outs, counts


_REF = {}


def _reference(gpu_lib, name, slabs, mode="host"):
    """Today's f64 interleaved calls on the input (whose values are exact in float32 and float64 alike)."""
    key = (name, slabs, mode)
    if key not in _REF:
        ch = _build(gpu_lib, name, slabs)
        x = _input(name, ch.channels, np.float64)
        if mode == "host":
            _REF[key] = _run_host(gpu_lib, ch, x, F64, F64, old_api=True)
        else:
            _REF[key] = (_submit(gpu_lib, ch, x, F64, F64, old_api=True), None)
        ch.close()
    return _REF[key]


@pytest.mark.parametrize("slabs", [1, 3])
@pytest.mark.parametrize("name", CHAINS)
def test_host_formats(gpu_lib, name, slabs):
    """The synchronous host call in all 16 format pairs: outputs bit-identical to today's call converted by numpy,
    padding untouched, one H2D and one D2H per shard and call, and the plain call's launches plus one edge kernel per
    converted side and shard (none for f64 interleaved on both sides, which is the plain call exactly)."""
    for in_fmt, out_fmt in PAIRS:
        want, ref_counts = _reference(gpu_lib, name, slabs)
        ch = _build(gpu_lib, name, slabs)
        S = ch.n_shards
        x = _input(name, ch.channels, _dtype(in_fmt))
        got, counts = _run_host(gpu_lib, ch, x, in_fmt, out_fmt, old_api=False)
        ch.close()
        what = (name, slabs, _name(in_fmt), _name(out_fmt))
        assert [g.shape[0] for g in got] == [w.shape[0] for w in want], what
        for k, (g, w) in enumerate(zip(got, want)):
            _same(g, _cast(w, out_fmt), what + (k,))
        n_calls = len(SIZES)
        for k, ((h2d, d2h, launches), (rh2d, rd2h, rlaunches), w) in enumerate(zip(counts, ref_counts, want)):
            assert (h2d, d2h) == (rh2d, rd2h), (what, k)
            if k < n_calls:
                assert h2d == S and d2h == (S if w.shape[0] else 0), (what, k, h2d, d2h)
            extra = S * ((k < n_calls and in_fmt != F64) + (out_fmt != F64 and w.shape[0] > 0))
            assert launches == rlaunches + extra, (what, k, launches, rlaunches)


def _submit(gpu_lib, ch, x, in_fmt, out_fmt, old_api):
    """Every call of SIZES * 2 submitted before any is waited for (more tickets than the ring of 8 holds): outputs."""
    sizes = SIZES + SIZES[:4]
    x = np.concatenate([x, x[:sum(SIZES[:4])] * 0.5])
    bufs, pos = [], 0
    for f in sizes:
        bi, bo = Buf(in_fmt, ch.channels, f), Buf(out_fmt, ch.channels, max(ch.max_out_frames(f), f, 1))
        bi.put(x[pos:pos + f])
        if old_api:
            n, t = ch.submit_raw(f, bi.ptr, bo.ptr)
        else:
            n, t = ch.submit_io_raw(f, bi.ptr, in_fmt, bi.stride, bo.ptr, out_fmt, bo.stride)
        bufs.append((bi, bo, n))
        pos += f
    ch.wait(t)
    for bi, bo, n in bufs:
        assert bo.guards_kept(n)
    return [bo.get(n) for _, bo, n in bufs]


@pytest.mark.parametrize("name", ["gain", "fir_p_multi", "resample_up", "combo"])
def test_submit_formats(gpu_lib, name):
    """submit/wait on 3 slabs with 12 blocks outstanding in all 16 pairs: bit-identical to today's submit_raw."""
    for in_fmt, out_fmt in PAIRS:
        want, _ = _reference(gpu_lib, name, 3, mode="submit")
        ch = _build(gpu_lib, name, 3)
        got = _submit(gpu_lib, ch, _input(name, ch.channels, _dtype(in_fmt)), in_fmt, out_fmt, old_api=False)
        ch.close()
        assert len(got) == len(want)
        for k, (g, w) in enumerate(zip(got, want)):
            _same(g, _cast(w, out_fmt), (name, _name(in_fmt), _name(out_fmt), k))


# ------------------------------------------------------------------------------------------------------------
# Mode D
# ------------------------------------------------------------------------------------------------------------
def _dev_buf(fmt, n, frames, odd):
    """A canary-filled device buffer for a shard of n channels: (tensor, element offset of the slab, stride); f32 slabs
    start one element past a 16-byte boundary when `odd`."""
    import torch
    dt = torch.float32 if fmt & F32 else torch.float64
    off = 8 + (1 if odd and fmt & F32 else 0)
    stride = frames + PAD if fmt & PLANAR else 0
    size = n * stride if fmt & PLANAR else (frames + PAD) * n
    t = torch.empty(off + size + 8, dtype=dt, device="cuda")
    t.view(_int_type(t)).fill_(CANARY[_dtype(fmt)])   # both canaries are positive as signed integers
    return t, off, stride


def _int_type(t):
    import torch
    return torch.int64 if t.dtype == torch.float64 else torch.int32


def _slab(t, off, fmt, n, frames, stride):
    """The [frames, n] view of a shard's samples in a buffer of _dev_buf."""
    if fmt & PLANAR:
        return t[off:off + n * stride].view(n, stride)[:, :frames].t()
    return t[off:off + frames * n].view(frames, n)


def _run_device(gpu_lib, ch, x, in_fmt, out_fmt, odd, in_place=False, sizes=SIZES):
    """The calls of `sizes` (reset before RESET_AT) shard by shard on a new non-blocking stream, a _sleep before each:
    outputs per call.  Asserts guards, the input's bits (out of place) and d_in's alignment."""
    import torch
    shards = [ch.shard_info(s) for s in range(ch.n_shards)]
    s = torch.cuda.Stream()
    outs, checks, pos = [], [], 0
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    for i, f in enumerate(sizes):
        if i == RESET_AT:
            torch.cuda.synchronize()
            ch.reset()
        mo = max(ch.max_out_frames(f), f if in_place else 0, 1)
        parts, got = [], set()
        with torch.cuda.stream(s):
            for k, (_, b, n) in enumerate(shards):
                ti, oi, si = _dev_buf(in_fmt, n, max(f, mo) if in_place else f, odd)
                _slab(ti, oi, in_fmt, n, f, si).copy_(xd[pos:pos + f, b:b + n])
                if in_place:
                    to, oo, so = ti, oi, si
                else:
                    to, oo, so = _dev_buf(out_fmt, n, mo, odd)
                snap = ti.clone()
                torch.cuda._sleep(SLEEP_CYCLES)
                esz_i, esz_o = ti.element_size(), to.element_size()
                m = ch.run_device_io(k, f, ti.data_ptr() + esz_i * oi, in_fmt, si, to.data_ptr() + esz_o * oo, out_fmt, so, s.cuda_stream)
                got.add(m)
                parts.append((to, oo, so, n, ti, snap))
        assert len(got) == 1, got
        m = got.pop()
        with torch.cuda.stream(s):
            cols = []
            for to, oo, so, n, ti, snap in parts:
                out = _slab(to, oo, out_fmt, n, m, so).clone()
                cols.append(out)
                # everything but the returned rows keeps the canary; d_in keeps its bits unless in place
                mask = torch.ones_like(to, dtype=torch.bool)
                _slab(mask, oo, out_fmt, n, m, so).fill_(False)
                if in_place:
                    checks.append((to.view(_int_type(to))[mask] == snap.view(_int_type(snap))[mask]).all())
                else:
                    checks.append((to.view(_int_type(to))[mask] == CANARY[_dtype(out_fmt)]).all())
                    checks.append((ti.view(_int_type(ti)) == snap.view(_int_type(snap))).all())
            outs.append(torch.cat(cols, dim=1))
        pos += f
    torch.cuda.synchronize()
    for k, ok in enumerate(checks):
        assert bool(ok), ("a Mode D call wrote outside its returned rows or changed d_in", k, _name(in_fmt), _name(out_fmt))
    return [o.cpu().numpy() for o in outs]


@pytest.mark.parametrize("slabs", [1, 3])
@pytest.mark.parametrize("name", CHAINS)
def test_device_formats(gpu_lib, name, slabs):
    """Mode D in all 16 pairs, shard by shard, on a non-default stream with a _sleep ahead of every call, f32 rows on
    4-byte (not 16-byte) boundaries: bit-identical to today's host call converted by numpy, canary intact around the
    returned rows, d_in unchanged."""
    for in_fmt, out_fmt in PAIRS:
        want, _ = _reference(gpu_lib, name, slabs)
        ch = _build(gpu_lib, name, slabs)
        got = _run_device(gpu_lib, ch, _input(name, ch.channels, _dtype(in_fmt)).astype(_dtype(in_fmt)), in_fmt, out_fmt, odd=True)
        ch.close()
        for k, (g, w) in enumerate(zip(got, want[:len(SIZES)])):
            _same(g, _cast(w, out_fmt), (name, slabs, _name(in_fmt), _name(out_fmt), k))


@pytest.mark.parametrize("fmt", FORMATS, ids=_name)
@pytest.mark.parametrize("name", ["biquad10", "fir_p_short"])
def test_device_in_place(gpu_lib, name, fmt):
    """Mode D in place (same format and stride), on 16-byte-aligned rows: bit-identical, padding untouched."""
    want, _ = _reference(gpu_lib, name, 1)
    ch = _build(gpu_lib, name, 1)
    got = _run_device(gpu_lib, ch, _input(name, ch.channels, _dtype(fmt)), fmt, fmt, odd=False, in_place=True)
    ch.close()
    for k, (g, w) in enumerate(zip(got, want[:len(SIZES)])):
        _same(g, _cast(w, fmt), (name, _name(fmt), k))


# ------------------------------------------------------------------------------------------------------------
# the conversions themselves: ragged shapes and edge values
# ------------------------------------------------------------------------------------------------------------
FLT_MAX = float(np.finfo(np.float32).max)
SPECIALS = [0.0, -0.0, np.inf, -np.inf, np.nan, FLT_MAX, -FLT_MAX, 2.0 * FLT_MAX, -1e300, FLT_MAX * (1 + 2.0 ** -26),
            FLT_MAX * (1 + 2.0 ** -23), 1e-40, -1e-45, 1.4e-45, 5e-324, 1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24, 1 / 3.0]


def _edge_input(C, frames, seed):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((frames, C)) * 10.0 ** rng.integers(-50, 50, (frames, C))
    flat = x.reshape(-1)
    k = min(len(SPECIALS), flat.size)
    flat[rng.choice(flat.size, k, replace=False)] = SPECIALS[:k]
    return x


@pytest.mark.parametrize("C", [1, 2, 7, 256])
@pytest.mark.parametrize("frames", [1, 4097])
def test_conversions(gpu_lib, C, frames):
    """A chain without operators is the conversion alone: in all 16 pairs, host and Mode D (f32 rows on 4-byte and on
    16-byte boundaries), the output is numpy's conversion of the input bit for bit (NaN by isnan): +-0, +-Inf, NaN,
    subnormals, values beyond FLT_MAX (+-Inf) and just above it (rounded to FLT_MAX or Inf as numpy rounds), every
    tile edge of the planar transpose (1, 2, 7 and 256 channels, 1 and 4097 frames)."""
    import torch
    x64 = _edge_input(C, frames, C * 7 + frames)
    for in_fmt, out_fmt in PAIRS:
        xin = _cast(x64, in_fmt)
        want = _cast(xin.astype(np.float64), out_fmt)
        ch = gpu_lib.Chain(48000, C)
        bi, bo = Buf(in_fmt, C, frames), Buf(out_fmt, C, frames)
        bi.put(xin)
        n = ch.run_io_raw(frames, bi.ptr, in_fmt, bi.stride, bo.ptr, out_fmt, bo.stride)
        assert n == frames and bo.guards_kept(n)
        _same(bo.get(n), want, ("host", C, frames, _name(in_fmt), _name(out_fmt)))
        for odd in (False, True):
            got = _run_device(gpu_lib, ch, xin, in_fmt, out_fmt, odd, sizes=[frames])
            _same(got[0], want, ("device", odd, C, frames, _name(in_fmt), _name(out_fmt)))
        ch.close()
    torch.cuda.synchronize()


def test_subnormal_outputs(gpu_lib):
    """A gain of 1e-40 makes float32 subnormals of ordinary samples: they must come out exactly as numpy rounds them
    (a flush to zero would give 0)."""
    C, F = 5, 3000
    x = (np.random.default_rng(3).standard_normal((F, C))).astype(np.float32)
    for in_fmt in FORMATS:
        for out_fmt in (F32, F32 | PLANAR):
            ch = gpu_lib.Chain(48000, C).add_gain(1e-40)
            bi, bo = Buf(in_fmt, C, F), Buf(out_fmt, C, F)
            bi.put(x.astype(_dtype(in_fmt)))
            n = ch.run_io_raw(F, bi.ptr, in_fmt, bi.stride, bo.ptr, out_fmt, bo.stride)
            ch.close()
            want = (x.astype(np.float64) * 1e-40).astype(np.float32)
            assert (want != 0).mean() > 0.99 and (np.abs(want[want != 0]) < np.finfo(np.float32).tiny).all()
            _same(bo.get(n), want, (_name(in_fmt), _name(out_fmt)))


def test_nonfinite_stays_in_its_channel(gpu_lib):
    """NaN and +-Inf on one channel of a FIR chain in f32 planar: the other channels stay finite and bit-identical to
    today's call, and the poisoned channel matches it by isnan."""
    C, F = 4, 4096
    x = (np.random.default_rng(9).standard_normal((3 * F, C)) * 0.2).astype(np.float32)
    x[100, 2], x[5000, 2], x[9000, 2] = np.nan, np.inf, -np.inf
    ref = gpu_lib.Chain(44100, C).add_fir(_taps(3000, C, 2), block_hint=F)
    ch = gpu_lib.Chain(44100, C).add_fir(_taps(3000, C, 2), block_hint=F)
    for k in range(3):
        xb = x[k * F:(k + 1) * F]
        want = ref.run(xb.astype(np.float64))
        got = ch.run_io(np.ascontiguousarray(xb.T), planar=True)
        assert got.dtype == np.float32 and got.shape == (C, F)
        _same(got.T, want.astype(np.float32), k)
        assert np.isfinite(got[[0, 1, 3]]).all()
    ref.close()
    ch.close()


# ------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------
def test_refusals(gpu_lib):
    """Each refusal returns < 0 with its message before anything is enqueued (no copy, no launch), and the stream
    continued afterwards is bit-identical to a chain that never saw the bad calls."""
    import torch
    name = "combo"
    x = _input(name, 7, np.float32)
    good = _build(gpu_lib, name, 3)
    bad = _build(gpu_lib, name, 3)
    one = _build(gpu_lib, "fir_p_short", 1)
    f = 4096
    mo = bad.max_out_frames(f)
    assert mo > f + PAD
    bi = Buf(F32 | PLANAR, 7, f)          # stride f + PAD
    bi.put(x[:f])
    bo = Buf(F32 | PLANAR, 7, mo)         # stride mo + PAD
    bw = Buf(F32 | PLANAR, 7, mo)         # in place: a stride that fits both sides
    bw.put(x[:f])
    L = gpu_lib.lib()

    def host(in_fmt, in_stride, out_ptr, out_fmt, out_stride, buf=bi):
        return lambda: L.dspb200_chain_run_host_io(bad.h, f, buf.ptr, in_fmt, in_stride, out_ptr, out_fmt, out_stride)
    cases = [
        ("unknown format bits", -1, host(0x21, bi.stride, bo.ptr, F32 | PLANAR, bo.stride)),
        ("unknown format bits", -1, host(F32 | PLANAR, bi.stride, bo.ptr, F32 | 0x100, bo.stride)),
        ("interleaved input takes stride 0", -1, host(F32, 5, bo.ptr, F32 | PLANAR, bo.stride)),
        ("interleaved output takes stride 0", -1, host(F32 | PLANAR, bi.stride, bo.ptr, F32, 7)),
        ("planar input stride %d is shorter" % (f - 1), -1, host(F32 | PLANAR, f - 1, bo.ptr, F32 | PLANAR, bo.stride)),
        ("max_out_frames %d" % mo, -1, host(F32 | PLANAR, bi.stride, bo.ptr, F32 | PLANAR, mo - 1)),
        ("in place needs", -1, host(F32 | PLANAR, bw.stride, bw.ptr, F64 | PLANAR, bw.stride, buf=bw)),
        ("in place needs", -1, host(F32 | PLANAR, bw.stride, bw.ptr, F32 | PLANAR, bw.stride + 1, buf=bw)),
        ("unknown format bits", -1, lambda: L.dspb200_chain_submit_host_io(bad.h, f, bi.ptr, F32 | 0x40, bi.stride, bo.ptr, F32, 0, None)),
        ("max_out_frames", -2, lambda: L.dspb200_chain_drain_host_io(bad.h, f, bo.ptr, F32 | PLANAR, mo - 1)),
        ("unknown format bits", -2, lambda: L.dspb200_chain_drain_host_io(bad.h, f, bo.ptr, 0x2, 0)),
    ]
    for message, want_rc, call in cases:
        c0 = _counts(gpu_lib)
        rc = call()
        assert rc == want_rc and message in gpu_lib.last_error(), (message, rc, gpu_lib.last_error())
        assert _counts(gpu_lib) == c0, message
    assert bo.guards_kept(0) and bw.get(f).tobytes() == x[:f].tobytes()
    # Mode D: a misaligned f32 row, a planar stride below the frames, in place across formats, in place on a chain
    # whose last operator changes the frame count
    d = torch.zeros(8 * f + 64, dtype=torch.float32, device="cuda")
    p = d.data_ptr()
    dev_cases = [
        ("not aligned", one, (p + 2, F32, 0, p + 4096, F32, 0)),
        ("planar input stride 15 is shorter", one, (p, F32 | PLANAR, 15, p + 4096, F32 | PLANAR, 16)),
        ("in place needs", one, (p, F32, 0, p, F64, 0)),
        ("in-place call on a chain whose last operator changes the frame count", bad, (p, F32, 0, p, F32, 0)),
    ]
    for message, ch, (a, fa, sa, b, fb, sb) in dev_cases:
        c0 = _counts(gpu_lib)
        with pytest.raises(gpu_lib.DspB200Error, match=message):
            ch.run_device_io(0, 16, a, fa, sa, b, fb, sb, None)
        assert _counts(gpu_lib) == c0, message
    torch.cuda.synchronize()
    for ch in (good, bad):
        pos = 0
        outs = []
        for fr in SIZES:
            b1, b2 = Buf(F32 | PLANAR, 7, fr), Buf(F32, 7, max(ch.max_out_frames(fr), fr))
            b1.put(x[pos:pos + fr])
            n = ch.run_io_raw(fr, b1.ptr, F32 | PLANAR, b1.stride, b2.ptr, F32, 0)
            outs.append(b2.get(n))
            pos += fr
        ch.outs = outs
    for k, (g, w) in enumerate(zip(bad.outs, good.outs)):
        _same(g, w, ("after refusals", k))
    for ch in (good, bad, one):
        ch.close()


# ------------------------------------------------------------------------------------------------------------
# Python entry points
# ------------------------------------------------------------------------------------------------------------
def test_run_io_and_run_tensor(gpu_lib):
    """run_io keeps the dtype and layout of its input (and takes a wider `out`), run_tensor does the same for CUDA
    tensors on the current stream, drain_io returns the drain in the asked format; all match today's calls converted
    by numpy.  run_tensor refuses a multi-shard chain with a message."""
    import torch
    name = "resample_up"
    x = _input(name, 7, np.float32)
    want, _ = _reference(gpu_lib, name, 1)
    for dtype in (np.float32, np.float64):
        for planar in (False, True):
            ch = _build(gpu_lib, name, 1)
            pos, outs = 0, []
            for i, f in enumerate(SIZES):
                if i == RESET_AT:
                    ch.reset()
                xb = x[pos:pos + f].astype(dtype)
                if planar:
                    wide = np.full((7, f + 10), np.nan, dtype=dtype)
                    wide[:, :f] = xb.T
                    out = np.full((7, ch.max_out_frames(f) + 5), -7.0, dtype=dtype)
                    y = ch.run_io(wide[:, :f], planar=True, out=out)
                    assert y.base is out or y.base is out.base
                    assert (out[:, y.shape[1]:] == -7.0).all()
                    y = y.T
                else:
                    y = ch.run_io(xb)
                assert y.dtype == dtype
                outs.append(y.copy())
                pos += f
            while (y := ch.drain_io(1024, dtype=dtype, planar=planar)) is not None:
                outs.append(y.T if planar else y)
            ch.close()
            assert len(outs) == len(want)
            for k, (g, w) in enumerate(zip(outs, want)):
                _same(np.ascontiguousarray(g), _cast(w, F32 if dtype == np.float32 else F64), (dtype, planar, k))
    for dtype in (torch.float32, torch.float64):
        for planar in (True, False):
            ch = _build(gpu_lib, name, 1)
            s = torch.cuda.Stream()
            pos, outs = 0, []
            xt = torch.from_numpy(x).cuda()
            with torch.cuda.stream(s):
                for i, f in enumerate(SIZES):
                    if i == RESET_AT:
                        torch.cuda.synchronize()
                        ch.reset()
                    xb = xt[pos:pos + f].to(dtype)
                    xb = xb.t().contiguous() if planar else xb.contiguous()
                    torch.cuda._sleep(SLEEP_CYCLES)
                    y = ch.run_tensor(xb, planar=planar)
                    assert y.dtype == dtype and y.is_cuda
                    assert y.shape[0 if planar else 1] == 7
                    outs.append((y.t() if planar else y).clone())
                    pos += f
            torch.cuda.synchronize()
            ch.close()
            for k, (g, w) in enumerate(zip(outs, want)):
                _same(g.cpu().numpy(), _cast(w, F32 if dtype == torch.float32 else F64), (dtype, planar, k))
    ch = _build(gpu_lib, name, 3)
    with pytest.raises(gpu_lib.DspB200Error, match="single-shard"):
        ch.run_tensor(torch.zeros(7, 100, device="cuda"))
    ch.close()


def test_edge_profile(gpu_lib):
    """The edge kernels are timed under the name "edge"; an f64 interleaved call launches none."""
    ch = gpu_lib.Chain(48000, 4).add_gain(2.0)
    x = np.ones((1000, 4), dtype=np.float32)
    gpu_lib.profile_read("edge")
    gpu_lib.profile_enable(True)
    try:
        ch.run_io(x.astype(np.float64))
        assert gpu_lib.profile_read("edge")[1] == 0
        ch.run_io(x)
        ms, n = gpu_lib.profile_read("edge")
    finally:
        gpu_lib.profile_enable(False)
    ch.close()
    assert n == 2 and ms > 0, (ms, n)


def test_two_devices(gpu_lib):
    """Shards on two GPUs (skipped with one): every pair bit-identical to the same chain on two devices through today's
    call."""
    if gpu_lib.device_count() < 2:
        pytest.skip("one device")
    for name in ("fir_p_multi", "combo"):
        ref = _build(gpu_lib, name, 2, devices=[0, 1])
        want, _ = _run_host(gpu_lib, ref, _input(name, 7, np.float64), F64, F64, old_api=True)
        ref.close()
        for in_fmt, out_fmt in PAIRS:
            ch = _build(gpu_lib, name, 2, devices=[0, 1])
            got, _ = _run_host(gpu_lib, ch, _input(name, 7, _dtype(in_fmt)), in_fmt, out_fmt, old_api=False)
            ch.close()
            for k, (g, w) in enumerate(zip(got, want)):
                _same(g, _cast(w, out_fmt), (name, _name(in_fmt), _name(out_fmt), k))
