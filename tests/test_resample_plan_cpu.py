"""CPU tier: the resampler's host logic, dsp_b200/csrc/resample_plan.h, compiled with g++ alone.

resample_params() against oracle/restate.py's Resampler; RsPacing (the frames each call and drain poll emits, and the
first raw output index of each call) against accuracy.RsPacing; rs_launch() (the kernel, tile and warps per CTA of each
call) against accuracy.rs_expect_launch, which the GPU tests also check against describe().
"""
import ctypes

import numpy as np
import pytest

from accuracy import RS_RATIOS, RsPacing, header_lib, rs_expect_launch

DRIVER = r"""
#include "resample_plan.h"
using namespace dspb200;
extern "C" {
// n, d, m, in_len, out_len, out_delay, sinc_len; returns resample_params()'s code
int params(int fs_in, int fs_out, double bw, long *out)
{
	ResampleParams p;
	const int e = resample_params(fs_in, fs_out, bw, &p);
	if (!e) { out[0] = p.n; out[1] = p.d; out[2] = p.m; out[3] = p.in_len; out[4] = p.out_len; out[5] = p.out_delay; out[6] = p.sinc_len; }
	return e;
}
void *pace_new(int fs_in, int fs_out, double bw)
{
	ResampleParams p;
	return resample_params(fs_in, fs_out, bw, &p) ? nullptr : new RsPacing{p};
}
void pace_free(void *s) { delete (RsPacing *) s; }
void pace_reset(void *s) { ((RsPacing *) s)->reset(); }
long pace_run(void *s, long frames, long *first)
{
	const RsCall c = ((RsPacing *) s)->run(frames);
	*first = c.first;
	return c.frames;
}
// one poll of ResampleOp::drain2's bookkeeping: -1 when dry, else the frames it returns; *ran: the frames its run emitted
long pace_drain(void *s, long frames, long *first, long *ran)
{
	RsPacing *p = (RsPacing *) s;
	if (p->drain_dry()) return -1;
	const RsCall c = p->run(frames);
	*first = c.first;
	*ran = c.frames;
	return (c.frames < 0) ? -2 : p->drain_trim(c.frames);
}
// tile, warps, depth, minb, Q, channels; returns the kernel's name
const char *launch(int C, long oframes, int sms, int force_tile, int *out)
{
	const RsLaunch L = rs_launch(C, oframes, sms, force_tile);
	out[0] = L.tile; out[1] = L.warps; out[2] = L.depth; out[3] = L.minb; out[4] = L.Q; out[5] = L.channels;
	return L.kernel;
}
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    lib = header_lib(tmp_path_factory.mktemp("resample_plan"), "resampleplan", DRIVER)
    lib.params.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_double, ctypes.POINTER(ctypes.c_long)]
    lib.pace_new.restype = ctypes.c_void_p
    lib.pace_new.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_double]
    lib.pace_free.argtypes = lib.pace_reset.argtypes = [ctypes.c_void_p]
    lib.pace_run.restype = ctypes.c_long
    lib.pace_run.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.POINTER(ctypes.c_long)]
    lib.pace_drain.restype = ctypes.c_long
    lib.pace_drain.argtypes = [ctypes.c_void_p, ctypes.c_long, ctypes.POINTER(ctypes.c_long), ctypes.POINTER(ctypes.c_long)]
    lib.launch.restype = ctypes.c_char_p
    lib.launch.argtypes = [ctypes.c_int, ctypes.c_long, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    return lib


def _rates_id(r):
    return "%d-%d" % r


def _params(lib, fi, fo, bw):
    out = (ctypes.c_long * 7)()
    e = lib.params(fi, fo, bw, out)
    return e, dict(zip(("n", "d", "m", "in_len", "out_len", "out_delay", "sinc_len"), out))


@pytest.mark.parametrize("rates", RS_RATIOS, ids=_rates_id)
def test_params(lib, rates):
    """Every field against restate.Resampler at bandwidths 0.7, 0.939 (also as 0, the default), 0.99 and 0.999."""
    from oracle import restate
    fi, fo = rates
    for bw in (0.7, 0.939, 0.99, 0.999):
        r = restate.Resampler(fi, fo, 1, bw=bw)
        want = dict(n=r.n, d=r.d, m=r.m, in_len=r.in_len, out_len=r.out_len, out_delay=r.out_delay, sinc_len=r.sinc_fr_len - 1)
        assert _params(lib, fi, fo, bw) == (0, want), (bw, want)
    assert _params(lib, fi, fo, 0.0) == _params(lib, fi, fo, 0.939)


@pytest.mark.parametrize("fi,fo,bw,code", [(0, 48000, 0.939, 1), (48000, 0, 0.939, 1), (-44100, 48000, 0.939, 1),
                                           (48000, 48000, 0.939, 1), (44100, 48000, 0.6999, 2), (44100, 48000, 0.9991, 2),
                                           (44100, 48000, 1.0, 2), (44100, 48000, -0.939, 2), (44100, 48000, float("nan"), 2)])
def test_params_refused(lib, fi, fo, bw, code):
    """Rates that are not positive or equal (RS_BAD_RATES), bandwidths outside [0.7, 0.999] (RS_BAD_BANDWIDTH)."""
    assert _params(lib, fi, fo, bw)[0] == code


@pytest.mark.parametrize("rates", RS_RATIOS, ids=_rates_id)
def test_pacing(lib, rates):
    """Seeded ragged calls (1 frame, in_len - 1, in_len, in_len + 1, 4096 and random sizes), reset() in the middle,
    drains polled 1, 7, 4096 frames or a random size at a time until dry, and after another reset() a stream whose
    drain is dry at once (the drain counters survive reset(), as in the reference): every call's and poll's count
    against accuracy.RsPacing, and the first raw output index of each call that emits frames is out_delay plus the
    frames emitted since the last reset()."""
    fi, fo = rates
    want = RsPacing(fi, fo)
    L, delay = want.in_len, want.out_delay
    rng = np.random.default_rng(fi * 7 + fo)

    def calls():
        sizes = [1, L - 1, L, L + 1, 4096, 1, 1]
        sizes += [int(v) for v in rng.integers(1, 3 * L + 2, 12)] + [int(v) for v in rng.integers(1, 64, 12)]
        rng.shuffle(sizes)
        return sizes

    s = lib.pace_new(fi, fo, 0.939)
    first, ran = ctypes.c_long(), ctypes.c_long()
    try:
        emitted, drains = 0, []
        for step in ("run", "reset", "run", "drain", "reset", "run", "drain"):
            if step == "reset":
                lib.pace_reset(s)
                want.reset()
                emitted = 0
            elif step == "run":
                for f in calls():
                    got = lib.pace_run(s, f, ctypes.byref(first))
                    assert got == want.run(f), (step, f)
                    if got:
                        assert first.value == delay + emitted, (f, first.value, emitted)
                    emitted += got
            else:
                polls = 0
                while True:
                    f = int(rng.choice([1, 7, 4096, int(rng.integers(1, 2 * L))]))
                    got = lib.pace_drain(s, f, ctypes.byref(first), ctypes.byref(ran))
                    w = want.drain(f)
                    assert got == (-1 if w is None else w), (f, got, w)
                    if got < 0:
                        break
                    if ran.value:
                        assert first.value == delay + emitted, (f, first.value, emitted)
                    emitted += ran.value
                    polls += 1
                drains.append(polls)
        assert drains[0] > 0 and drains[1] == 0, drains
    finally:
        lib.pace_free(s)


LAUNCH_CHANNELS = list(range(1, 301)) + [512, 1024, 2048]


def _oframes_grid(C, sms):
    """1 .. 4 sms 32 output frames: a coarse grid, and both sides of each warps threshold (the last call size whose
    output tiles leave too few CTAs per SM, and the first that leaves enough)."""
    top = 4 * sms * 32
    grid = {1, 31, 32, 33, 64, 65, top - 1, top}
    grid.update(int(v) for v in np.geomspace(1, top, 24))
    for w, per_sm in ((4, 3), (2, 2)):
        cols = -(-C // (32 * w))
        tiles = -(-per_sm * sms // cols)          # fewest output tiles of 32 frames that reach per_sm CTAs per SM
        for o in (32 * (tiles - 1), 32 * (tiles - 1) + 1):
            if 1 <= o <= top:
                grid.add(o)
    return sorted(grid)


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_launch(lib, sms):
    """rs_launch() against rs_expect_launch, field by field, for every C in 1..300, 512, 1024 and 2048, every
    DSP_B200_RS_TILE from -1 to 8 and the call sizes of _oframes_grid."""
    out = (ctypes.c_int * 6)()
    keys = ("tile", "warps", "depth", "minb", "Q", "channels")
    seen = set()
    for C in LAUNCH_CHANNELS:
        grid = _oframes_grid(C, sms)
        for force in range(-1, 9):
            for o in grid:
                kernel = lib.launch(C, o, sms, force, out).decode()
                got = dict(zip(keys, out), kernel=kernel)
                want = rs_expect_launch(C, force, o, sms)
                assert got == want, (C, force, o, got, want)
                seen.add((got["tile"], got["warps"]))
    # every tile, and every warps choice of each tensor-core tile, was reached
    assert seen == {(1, 4), (2, 2), (3, 4)} | {(t, w) for t in (4, 5, 6, 7) for w in (1, 2, 4)}, seen
