"""Extended-precision references and one error metric for the accuracy tests (test code only; the product never
imports it).

FIR: `exact_conv` is the exact linear convolution of dyadic signals.  x = k 2^-12 with |k| <= 2^11 and
h = j 2^-S with |j| <= 2^12, so every output sample is an integer multiple of 2^-(12+S) whose numerator needs
about 23 + log2(taps) bits: at 131072 taps and beyond it is still far inside the 53 bits of a double.  The
FP64 FFT convolution of the integer numerators is then within a small fraction of a unit of the exact
integers, and rounding to the grid recovers them exactly.

Biquad: `biquad_truth` runs the same double coefficients through scipy's lfilter in 80-bit long double;
`bq_expect_launch` restates the kernel form each call gets.

Resample: `resample_taps_truth` is the tap table G of the polyphase form (resample.cu header) in long double, built
from the reference's own sinc samples; `resample_truth` evaluates the emitted stream from it in long double, and
`RsPacing` / `rs_counts` replay the per-call frame counts in integers.

Errors are reported as nerr = rms(got - want) / scale (and nmax with the max): for FIR, scale = rms(x) ||h||_2
per channel, for resample rms(x) ||G|| per channel (`rs_nerr`), elsewhere scale = rms(want).
"""
import ctypes
import os
import subprocess
from contextlib import contextmanager

import numpy as np

X_SHIFT = 12       # x = k 2^-12
X_MAX = 1 << 11    # |k| <= 2^11
H_MAX = 1 << 12    # |j| <= 2^12
U = 2.0 ** -53     # unit roundoff of FP64


def dyadic_signal(rng, frames, channels, amp=0.5):
    """Uniform white noise of peak `amp` (<= 0.5) on the grid k 2^-12."""
    kmax = min(int(amp * (1 << X_SHIFT)), X_MAX)
    return rng.integers(-kmax, kmax + 1, size=(frames, channels)).astype(np.float64) * 2.0 ** -X_SHIFT


def dyadic_taps(h, shift):
    """Round `h` (any shape; its peak is scaled to 1) to the grid j 2^-shift, |j| <= 2^12."""
    h = np.asarray(h, dtype=np.float64)
    peak = np.max(np.abs(h))
    return np.round(h / peak * H_MAX) * 2.0 ** -shift


def _numerators(a, shift, what):
    k = np.asarray(a, dtype=np.float64) * 2.0 ** shift
    assert np.array_equal(k, np.round(k)), "%s is not on the 2^-%d grid" % (what, shift)
    return k


def exact_conv(x, h, h_shift, selector=None, latency=0):
    """Exact linear convolution of dyadic x [frames, C] with dyadic taps h [T] or [T, fc] (column k -> k-th
    selected channel), delayed by `latency` frames, first `frames` frames: the stream restate.fir_stream describes.
    Unselected channels pass through.  Fails when the FP64 FFT lands more than 0.05 units off the output grid,
    i.e. when the operands exceed the bit budget."""
    x = np.asarray(x, dtype=np.float64)
    frames, C = x.shape
    h = np.asarray(h, dtype=np.float64)
    if h.ndim == 1:
        h = h[:, None]
    kx = _numerators(x, X_SHIFT, "x")
    kh = _numerators(h, h_shift, "h")
    T = h.shape[0]
    nfft = 1
    while nfft < frames + T:
        nfft *= 2
    y = np.zeros((frames, C))
    sel = [True] * C if selector is None else [bool(s) for s in selector]
    cols = [c for c in range(C) if sel[c]]
    for c in range(C):
        if not sel[c]:
            y[:, c] = x[:, c]
    Hf = np.fft.rfft(kh, nfft, axis=0)
    n_keep = max(frames - latency, 0)
    for k, c in enumerate(cols):
        full = np.fft.irfft(np.fft.rfft(kx[:, c], nfft) * Hf[:, 0 if h.shape[1] == 1 else k], nfft)[:n_keep]
        r = np.round(full)
        dev = np.max(np.abs(full - r), initial=0.0)
        assert dev <= 0.05, "FFT result %.3g units off the grid: operands exceed the bit budget" % dev
        y[latency:, c] = r * 2.0 ** -(X_SHIFT + h_shift)
        if latency:
            y[:latency, c] = 0.0
    return y


def fir_scale(x, h, selector=None):
    """Per selected channel: rms(x_c) ||h_c||_2 (list, one entry per selected channel)."""
    x = np.asarray(x, dtype=np.float64)
    h = np.asarray(h, dtype=np.float64)
    if h.ndim == 1:
        h = h[:, None]
    cols = [c for c in range(x.shape[1]) if selector is None or selector[c]]
    return np.array([np.sqrt(np.mean(x[:, c] ** 2)) * np.linalg.norm(h[:, 0 if h.shape[1] == 1 else k])
                     for k, c in enumerate(cols)]), cols


def fir_nerr(got, want, x, h, selector=None):
    """(worst normalized RMS, worst normalized max) over the selected channels."""
    scale, cols = fir_scale(x, h, selector)
    d = np.asarray(got, dtype=np.float64)[:, cols] - np.asarray(want, dtype=np.float64)[:, cols]
    return float(np.max(np.sqrt(np.mean(d * d, axis=0)) / scale)), float(np.max(np.max(np.abs(d), axis=0) / scale))


def nerr(got, want, scale=None):
    """(rms(got - want) / scale, max|got - want| / scale); scale defaults to rms(want)."""
    d = np.asarray(got, dtype=np.float64) - np.asarray(want, dtype=np.float64)
    w = np.asarray(want, dtype=np.float64)
    if scale is None:
        scale = float(np.sqrt(np.mean(w * w)))
    return float(np.sqrt(np.mean(d * d))) / scale, float(np.max(np.abs(d), initial=0.0)) / scale


def biquad_truth(x, coefs):
    """x [frames, C]; coefs [S, 5] or [S, C, 5] (double).  The cascade in 80-bit long double: per stage,
    lfilter(b = c0..c2, a = [1, c3, c4]).  Returns long double."""
    from scipy.signal import lfilter
    y = np.asarray(x, dtype=np.float64).astype(np.longdouble)
    coefs = np.asarray(coefs, dtype=np.float64)
    if coefs.ndim == 2:
        coefs = np.repeat(coefs[:, None, :], y.shape[1], axis=1)
    for st in range(coefs.shape[0]):
        for c in range(y.shape[1]):
            k = coefs[st, c].astype(np.longdouble)
            y[:, c] = lfilter(k[:3], np.array([1.0, k[3], k[4]], dtype=np.longdouble), y[:, c])
    return y


BQ_TBL = 70   # doubles per channel and stage: 5 coefficients and a pad, 6 matrices M^(16 2^r), T, T^-1, G (2 x 16)


def bq_expect_launch(C, S, frames, force_ch=None, force_split=None):
    """The launch of a biquad call of `frames` frames on C channels and S stages, with DSP_B200_BQ_CH=`force_ch` and
    DSP_B200_BQ_SPLIT=`force_split` (None: unset) -- bq_launch() of dsp_b200/csrc/biquad_plan.h, restated.  Two
    channels per CTA unless the knob asks for 4, or for anything but 0, 2 and 4, which runs one.  The split form (two
    8-warp CTAs per channel pair, one launch per 4096 frames) runs on pairs only: on calls of at most 2048 frames, or as
    a non-negative DSP_B200_BQ_SPLIT says (0: never, else always).  The others take 16 warps (8 on one channel per
    CTA) and one launch.  smem: the CTA's channel tables."""
    ch = 2 if force_ch in (None, 0, 2) else 4 if force_ch == 4 else 1
    split = ch == 2 and (frames <= 2048 if force_split is None or force_split < 0 else force_split != 0)
    span = 4096 if split else frames
    return dict(ch=ch, split=int(split), threads=32 * (8 if split or ch == 1 else 16), grid=-(-C // ch),
                smem=ch * S * BQ_TBL * 8, span=span, launches=-(-frames // span))


def biquad_err(got, truth):
    """rms(got - truth) in long double, as a float."""
    d = np.asarray(got, dtype=np.float64).astype(np.longdouble) - truth
    return float(np.sqrt(np.mean(d * d)))


def biquad_within_ref(got, x, coefs, truth=None, ref64=None):
    """Per channel: err_gpu <= max(4 err_ref64, 64 u rms(truth)), both errors against biquad_truth, err_ref64 that of
    the reference's own FP64 recurrence (restate.biquad_cascade, or `ref64`: the reference library's output of the
    same stream).  `truth` may be given when it is already known.  Returns per channel (err_gpu, err_ref64, ratio to
    the bound), errors relative to rms(truth); asserts the bound."""
    from oracle import restate
    if truth is None:
        truth = biquad_truth(x, coefs)
    if ref64 is None:
        ref64 = restate.biquad_cascade(x, coefs)
    out = []
    for c in range(x.shape[1]):
        t = truth[:, c]
        e_gpu, e_ref = biquad_err(got[:, c], t), biquad_err(ref64[:, c], t)
        scale = float(np.sqrt(np.mean(t * t)))
        bound = max(4 * e_ref, 64 * U * scale)
        out.append((e_gpu / scale, e_ref / scale, e_gpu / bound))
        assert e_gpu <= bound, (c, e_gpu / scale, e_ref / scale)
    return out


# the ratios of test_gpu_parity.test_resample_ratios: large n (640/147), sinc_os = 1 (2:1, 1:2), 1:6 and 6:1
RS_RATIOS = [(44100, 48000), (48000, 44100), (48000, 96000), (96000, 48000), (44100, 32000), (44100, 96000),
             (44100, 192000), (192000, 44100), (96000, 44100), (88200, 44100), (44100, 88200), (48000, 8000),
             (8000, 48000), (11025, 48000), (8000, 44100)]


def resample_taps_truth(fs_in, fs_out, bw=0.939):
    """The resampler's tap table G [n, in_len] in long double: G[ph][t] = g(ph + t n) with
        g(tau) = 1/(2 in_len) [S_0 + 2 sum_{k=1}^{K-1} Re(S_k e^{i th k tau}) + Re(S_K e^{i th K tau})],
    th = 2 pi / Pd, Pd = 2 in_len n, K = sinc_len, S = DFT_{2K} of the reference's windowed sinc (resample.cu header).
    That sum is a real inverse DFT of length Pd whose bins 0..K-1 hold S_k and bin K holds S_K / 2 -- or S_K itself
    when K is the Nyquist bin Pd / 2 (ratios 1:m and m:1), which the inverse transform does not double."""
    from oracle import restate
    r = restate.Resampler(fs_in, fs_out, 1, bw=bw)
    return taps_from_sinc(r.sinc, r.n, r.in_len)


def taps_from_sinc(sinc, n, in_len):
    """resample_taps_truth for any 2K-point real array `sinc` (K = len(sinc) / 2)."""
    K = len(sinc) // 2
    S = np.fft.rfft(np.asarray(sinc, dtype=np.float64).astype(np.longdouble))
    Pd = 2 * in_len * n
    B = np.zeros(Pd // 2 + 1, dtype=np.clongdouble)
    B[:K] = S[:K]
    B[K] = S[K] if 2 * K == Pd else S[K] / 2
    g = np.fft.irfft(B, Pd) * (np.longdouble(Pd) / (2 * in_len))
    return g[np.arange(n)[:, None] + np.arange(in_len)[None, :] * n]


def taps_norm(G):
    """||G|| = sqrt(mean over phases of sum_t G[ph][t]^2): the gain of the resampler on white noise."""
    G = np.asarray(G, dtype=np.float64)
    return float(np.sqrt(np.mean(np.sum(G * G, axis=1))))


def resample_truth(x, fs_in, fs_out, bw, n_out, rows=None, G=None):
    """The emitted stream of the resampler on x [frames, C] (zero before the stream and after its end, which is what
    the drain feeds): y[q] = sum_t G[(m d) mod n][t] x[floor(m d / n) - t], m = out_delay + q, for q < n_out, or
    only for the emitted indices in `rows`.  Long double, in chunks of outputs so that memory stays bounded."""
    from oracle import restate
    r = restate.Resampler(fs_in, fs_out, 1, bw=bw)
    if G is None:
        G = resample_taps_truth(fs_in, fs_out, bw)
    x = np.asarray(x, dtype=np.float64)
    N, C = x.shape
    q = np.arange(n_out) if rows is None else np.asarray(rows, dtype=np.int64)
    m = r.out_delay + q
    ph, ih = (m * r.d) % r.n, (m * r.d) // r.n
    # x with in_len zero rows in front and zeros past the end: input row i lives at i + in_len
    hi = int(ih.max(initial=0)) + 1
    xp = np.zeros((r.in_len + max(hi, N), C), dtype=np.longdouble)
    xp[r.in_len:r.in_len + N] = x
    t = np.arange(r.in_len)
    y = np.zeros((q.size, C), dtype=np.longdouble)
    step = max(1, (1 << 21) // (r.in_len * C))
    for a in range(0, q.size, step):
        idx = (ih[a:a + step] + r.in_len)[:, None] - t[None, :]
        y[a:a + step] = np.einsum("qt,qtc->qc", G[ph[a:a + step]], xp[idx])
    return y


class RsPacing:
    """The resampler's per-call frame counts in integers: resample.c:91-151 (run), :154-161 (reset, which leaves the
    drain counters alone) and :163-188 (drain2).  drain() returns None where the library reports a dry drain."""

    def __init__(self, fs_in, fs_out, bw=0.939):
        from oracle import restate
        r = restate.Resampler(fs_in, fs_out, 1, bw=bw)
        self.n, self.d, self.in_len, self.out_len, self.out_delay = r.n, r.d, r.in_len, r.out_len, r.out_delay
        self.in_buf_pos = self.out_buf_pos = self.has_output = 0
        self.is_draining = self.drain_pos = self.drain_frames = 0

    def _max_out(self, frames):
        v = frames * self.n
        return v // self.d + (1 if v % self.d else 0)

    def run(self, frames):
        mo, i, o = self._max_out(frames), 0, 0
        while i < frames:
            take = min(self.in_len - self.in_buf_pos, frames - i)
            self.in_buf_pos += take
            i += take
            if self.has_output:
                e = min(self.out_len - self.out_buf_pos, mo - o)
                self.out_buf_pos += e
                o += e
            if self.in_buf_pos == self.in_len and (not self.has_output or self.out_buf_pos == self.out_len):
                self.in_buf_pos = self.out_buf_pos = 0
                if not self.has_output:
                    self.out_buf_pos = self.out_delay
                    self.has_output = 1
        return o

    def reset(self):
        self.in_buf_pos = self.out_buf_pos = self.has_output = 0

    def drain(self, frames):
        if not self.has_output and self.in_buf_pos == 0:
            return None
        if not self.is_draining:
            if self.has_output:
                self.drain_frames += self.out_delay + self.out_len - self.out_buf_pos
            self.drain_frames += self._max_out(self.in_buf_pos)
            self.is_draining = 1
        if self.drain_pos >= self.drain_frames:
            return None
        o = self.run(frames)
        self.drain_pos += o
        return o - max(self.drain_pos - self.drain_frames, 0)


def rs_counts(fs_in, fs_out, sizes, drain_block=None, bw=0.939):
    """(per-call frame counts of calls of `sizes` frames, counts of the drain polls of `drain_block` frames that
    follow until the drain is dry; [] without a drain)."""
    p = RsPacing(fs_in, fs_out, bw)
    counts = [p.run(int(f)) for f in sizes]
    drains = []
    while drain_block:
        o = p.drain(drain_block)
        if o is None:
            break
        drains.append(o)
    return counts, drains


def rs_nerr(got, want, x, G):
    """(worst normalized RMS, worst normalized max) over channels, scale = rms(x_c) ||G|| per channel: the size of the
    output white noise of that power would have, so a stopband input whose output is tiny still gives a meaningful
    figure."""
    x = np.asarray(x, dtype=np.float64)
    scale = np.sqrt(np.mean(x * x, axis=0)) * taps_norm(G)
    d = (np.asarray(got, dtype=np.float64).astype(np.longdouble) - np.asarray(want, dtype=np.longdouble)).astype(np.float64)
    return float(np.max(np.sqrt(np.mean(d * d, axis=0)) / scale)), float(np.max(np.max(np.abs(d), axis=0) / scale))


@contextmanager
def env(**kw):
    """Set (or, with None, unset) environment variables for the duration of the block; the library reads its plan-time
    switches with getenv() when an operator is planned."""
    old = {k: os.environ.get(k) for k in kw}
    for k, v in kw.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ------------------------------------------------------------------------------------------------------------
# FIR plans: the cases the GPU tests run and tests/test_fir_schedule_cpu.py and tests/test_fir_tiers_cpu.py plan on the CPU
# ------------------------------------------------------------------------------------------------------------
F4, F2 = 4096, 2048
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dsp_b200", "csrc")


def header_lib(tmp_dir, name, source):
    """Compile a C++ driver of a host-only header of dsp_b200/csrc (fir_plan.h, resample_plan.h, biquad_plan.h) with
    g++ alone (no CUDA); -> ctypes.CDLL."""
    src, so = tmp_dir / (name + ".cpp"), tmp_dir / ("lib%s.so" % name)
    src.write_text(source)
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC", "-I", CSRC, str(src), "-o", str(so)], check=True)
    return ctypes.CDLL(str(so))


def _single(B, P=None):
    return lambda p: len(p["levels"]) == 1 and p["levels"][0]["B"] == B and (P is None or p["levels"][0]["P"] == P)


# name: (call frames, taps, channels, block_hint, env, plan check)
FIR_CASES = {
    "multi_64": (64, 20000, 4, 0, {}, lambda p: len(p["levels"]) > 1 and p["levels"][0]["B"] == 64),
    "multi_300": (300, 50000, 4, 0, {}, lambda p: len(p["levels"]) > 1 and p["levels"][0]["B"] == 256),
    "multi_1000": (1000, 131072, 4, 0, {}, lambda p: len(p["levels"]) > 1 and p["levels"][0]["B"] == 512),
    "single_2048_t4": (F2, 131072, 8, F2, dict(DSP_B200_FIR_T=4), lambda p: _single(F2, 64)(p) and p["t_batch"] == 4),
    "single_2048_t6": (F2, 131072, 8, F2, dict(DSP_B200_FIR_T=6), lambda p: _single(F2, 64)(p) and p["t_batch"] == 6),
    "single_2048_t8": (F2, 131072, 8, F2, dict(DSP_B200_FIR_T=8), lambda p: _single(F2, 64)(p) and p["t_batch"] == 8),
    "single_4096_t4": (F4, 131072, 8, F4, dict(DSP_B200_FIR_T=4), lambda p: _single(F4, 32)(p) and p["t_batch"] == 4),
    "single_4096_t6": (F4, 131072, 8, F4, dict(DSP_B200_FIR_T=6), lambda p: _single(F4, 32)(p) and p["t_batch"] == 6),
    "single_4096_t8": (F4, 131072, 8, F4, dict(DSP_B200_FIR_T=8), lambda p: _single(F4, 32)(p) and p["t_batch"] == 8),
    "merge": (F4, 131072, 8, F4, dict(DSP_B200_FIR_MERGE=1), lambda p: _single(F4, 32)(p) and p["merge"] == 1),
    "pipe_4096": (F4, 131072, 8, F4, dict(DSP_B200_FIR_PIPE=1), lambda p: _single(F4, 32)(p) and p["pipe"] == 1),
    "pipe_2048": (F2, 70000, 8, F2, dict(DSP_B200_FIR_PIPE=1), lambda p: _single(F2)(p) and p["pipe"] == 1),
    "bulk_32768": (32768, 50000, 3, 32768, {}, lambda p: p["levels"] == [{"B": 8192, "P": 7}]),
}
for _far in (8, 12, 16):
    for _mode, _e in (("s", dict(DSP_B200_FIR_STAGGER=1)), ("u", dict(DSP_B200_FIR_STAGGER=0)),
                      ("u2", dict(DSP_B200_FIR_STAGGER=0, DSP_B200_FIR_FAR_CLASSES=2))):
        if _mode == "u2" and (_far // 2) % 4:
            continue   # two classes need t_far / 2 to be a multiple of t_batch (4): far tiers 8 and 16
        _e = dict(_e, DSP_B200_FIR_T2=_far, DSP_B200_FIR_T=4)
        _cls = 2 if _mode == "u2" else 1
        FIR_CASES["far%d_%s" % (_far, _mode)] = (
            F2, 131072, 8, F2, _e,
            (lambda far, stag, cls: lambda p: _single(F2, 64)(p) and p["t_far"] == far and p["stagger"] == stag
             and (stag or p["far_classes"] == cls))(_far, 1 if _mode == "s" else 0, _cls))


# Plan edges: every boundary fir_schedule() (fir_plan.h) draws, each case with the plan it must make.  A planner change that moves
# a case off its edge fails the plan assertion instead of quietly testing something else.
FIR_EDGES = {}


def _fir_plan(levels, **kw):
    """The describe() fields a case must show: levels [(B, P), ...]; tail_pf, t_batch, t_far, stagger, pipe and
    pipe_pf are 0 and bulk (blocks per bulk launch) is 1 unless given."""
    p = dict(levels=[{"B": B, "P": P} for B, P in levels], tail_pf=0, t_batch=0, t_far=0, stagger=0, bulk=1, pipe=0, pipe_pf=0)
    p.update(kw)
    return p


def _edge(group, name, taps, C, hint, plan, envs=None, sel=None, latency=0, rising=False, short=False, lead=(), call=None):
    """One case: `hint` is the block hint (level 0's B), `call` the frames per call of the whole-block pass (default
    B0), `lead` the first calls of the ragged pass, `rising` adds the rising family (threshold cases), `short` runs a
    stream shorter than the filter."""
    FIR_EDGES["%s/%s" % (group, name)] = dict(taps=taps, C=C, hint=hint, plan=plan, envs=envs or {}, sel=sel, latency=latency,
                                              rising=rising, short=short, lead=tuple(lead), call=call)


def _ladder(B0, last_P, top=4096):
    """Multi-level plans: level 0 (B0, P = 2), one partition on every level up to `top`, `last_P` on the last."""
    lv, B = [(B0, 2)], 2 * B0
    while B < top:
        lv.append((B, 1))
        B *= 2
    return lv + [(top, last_P)]


# single level, fused kernel, no tail: P = 1 up to T = B, P = 2 from one tap more
for _B in (64, F2, F4):
    for _T, _P in ((1, 1), (2, 1), (_B - 1, 1), (_B, 1), (_B + 1, 2), (2 * _B, 2)):
        _edge("fused", "B%d_T%d" % (_B, _T), _T, 3 if _B == 64 else 4 if _B == F2 else 5, _B, _fir_plan([(_B, _P)]))
# single level, tail thresholds: the tail from P = 3, the batch from P = 11, the stagger from P = 22
for _B in (F2, F4):
    for _k, _P, _kw, _thr in ((2, 3, {}, False), (10, 10, {}, False), (10, 11, dict(t_batch=4), True),
                              (21, 21, dict(t_batch=4), False), (21, 22, dict(t_batch=4, stagger=1), True)):
        _T = _k * _B + (_P - _k)
        _edge("tail", "B%d_P%d" % (_B, _P), _T, 4 if _B == F2 else 5, _B, _fir_plan([(_B, _P)], tail_pf=2, **_kw), rising=_thr)
_edge("tail", "B2048_P22_short", 21 * F2 + 1, 4, F2, _fir_plan([(F2, 22)], tail_pf=2, t_batch=4, stagger=1), short=True)
# far tier from P = 48 (whole launches: no stagger)
_edge("far", "P47", 47 * F2, 4, F2, _fir_plan([(F2, 47)], tail_pf=2, t_batch=4, stagger=1))
_edge("far", "P48", 47 * F2 + 1, 4, F2, _fir_plan([(F2, 48)], tail_pf=2, t_batch=4, t_far=8), rising=True)
# batch depths 6 and 8: the batch from P = 2 T + 3
for _tb, _k in ((6, 14), (8, 18)):
    _edge("depth", "T%d_P%d" % (_tb, _k), _k * F2, 4, F2, _fir_plan([(F2, _k)], tail_pf=2), envs=dict(DSP_B200_FIR_T=_tb))
    _edge("depth", "T%d_P%d" % (_tb, _k + 1), _k * F2 + 1, 4, F2, _fir_plan([(F2, _k + 1)], tail_pf=2, t_batch=_tb),
          envs=dict(DSP_B200_FIR_T=_tb), rising=True)
# pipeline kernel: it sums every partition itself (pipe_pf = P) until the batch starts at P = 11
for _B in (F2, F4):
    for _T, _P, _kw in ((2 * _B + 1, 3, dict(pipe_pf=3)), (3 * _B + 1, 4, dict(pipe_pf=4)), (10 * _B, 10, dict(pipe_pf=10)),
                        (10 * _B + 1, 11, dict(pipe_pf=6, t_batch=4))):
        _edge("pipe", "B%d_P%d" % (_B, _P), _T, 4, _B, _fir_plan([(_B, _P)], tail_pf=2, pipe=1, **_kw),
              envs=dict(DSP_B200_FIR_PIPE=1), rising=_P == 11)
# multi-level: an upper level holding one tap, the last level (4096) at P = 1 and 2 (the tail starts), 9 and 10 (the batch)
for _B0 in (64, 128, 256, 512, 1024):
    _C = {64: 3, 128: 4, 256: 5, 512: 4, 1024: 2}[_B0]
    _edge("multi", "B%d_T%d" % (_B0, 2 * _B0 + 1), 2 * _B0 + 1, _C, _B0, _fir_plan([(_B0, 2), (2 * _B0, 1)]))
    _edge("multi", "B%d_T%d" % (_B0, 4 * _B0), 4 * _B0, _C, _B0, _fir_plan([(_B0, 2), (2 * _B0, 1)]))
    _edge("multi", "B%d_T%d" % (_B0, 4 * _B0 + 1), 4 * _B0 + 1, _C, _B0, _fir_plan([(_B0, 2), (2 * _B0, 1), (4 * _B0, 1)]))
    _edge("multi", "B%d_T8192" % _B0, 8192, _C, _B0, _fir_plan(_ladder(_B0, 1)))
    _edge("multi", "B%d_T8193" % _B0, 8193, _C, _B0, _fir_plan(_ladder(_B0, 2), tail_pf=1), rising=True)
    _edge("multi", "B%d_T40960" % _B0, 40960, _C, _B0, _fir_plan(_ladder(_B0, 9), tail_pf=1))
    _edge("multi", "B%d_T40961" % _B0, 40961, _C, _B0, _fir_plan(_ladder(_B0, 10), tail_pf=1, t_batch=4), rising=True)
_edge("multi", "B256_T40961_short", 40961, 5, 256, _fir_plan(_ladder(256, 10), tail_pf=1, t_batch=4), short=True)
# the most levels a plan has (FIR_MAX_LEVELS = 8): seven upper levels feed `pend`
_edge("levels", "B64_cap8192", 131072, 2, 64, _fir_plan(_ladder(64, 15, top=8192), tail_pf=1, t_batch=4),
      envs=dict(DSP_B200_FIR_LEVEL_CAP=8192), rising=True)
# bulk form: off at P = 2, from P = 3; calls that bring 2, 3 + 5 frames, 4 and 9 blocks, then 1 and B - 1 frames
_BULK_LEAD = (1, 8191, 2 * 8192, 3 * 8192 + 5, 4 * 8192, 9 * 8192, 1, 8191)
for _hint, _nb in ((16384, 2), (32768, 4)):
    _edge("bulk", "hint%d_P2" % _hint, 16384, 3, _hint, _fir_plan([(8192, 2)]), lead=_BULK_LEAD, call=_hint)
    _edge("bulk", "hint%d_P3" % _hint, 16385, 3, _hint, _fir_plan([(8192, 3)], bulk=_nb), lead=_BULK_LEAD, call=_hint, rising=True)
    _edge("bulk", "hint%d_P10" % _hint, 10 * 8192, 3, _hint, _fir_plan([(8192, 10)], bulk=_nb), lead=_BULK_LEAD, call=_hint)
# FFT tiles: CPB = 256 / (B / 16) channels per CTA; one channel less and one more
for _B0, _cpb in ((64, 64), (128, 32), (256, 16), (512, 8), (1024, 4)):
    for _C in (_cpb - 1, _cpb + 1):
        _edge("cpb", "B%d_C%d" % (_B0, _C), 2 * _B0 + 1, _C, _B0, _fir_plan([(_B0, 2), (2 * _B0, 1)]))
_edge("cpb", "B2048_C3", F2 + 1, 3, F2, _fir_plan([(F2, 2)]))
# the fused kernel's cluster form takes 4 contiguous selected channels from an even one: an odd start and a
# count that is no multiple of 4 fall back to the per-channel form
for _B in (F2, F4):
    for _P in (2, 3):
        _pl = _fir_plan([(_B, _P)], tail_pf=2 if _P == 3 else 0)
        _T = (_P - 1) * _B + 1
        _edge("cluster", "B%d_P%d_sel1-4of6" % (_B, _P), _T, 6, _B, _pl, sel=[1 <= c <= 4 for c in range(6)])
        _edge("cluster", "B%d_P%d_sel2-9of10" % (_B, _P), _T, 10, _B, _pl, sel=[2 <= c <= 9 for c in range(10)])
        _edge("cluster", "B%d_P%d_all5" % (_B, _P), _T, 5, _B, _pl)
# fir's latency ring: latencies around the call size, calls shorter and longer than the latency, 1-frame calls
for _B0 in (64, F4):
    for _T in (17, 255):
        _pl = _fir_plan([(64, 1)] if _B0 == 64 and _T == 17 else [(64, 2), (128, 1)] if _B0 == 64 else [(F4, 1)])
        for _lat in sorted({1, 17, _B0 - 1, _B0, _B0 + 1, 3 * _B0 + 5}):
            _edge("latency", "B%d_T%d_lat%d" % (_B0, _T, _lat), _T, 3, _B0, _pl, latency=_lat,
                  lead=(1, 1, max(_lat - 1, 1), _lat, _lat + 1, 1, 2 * _lat + 3, 1, 1, 3 * _lat, 5),
                  envs=dict(DSP_B200_FIR_NO_REPLAN=1))   # calls longer than 2 B0 keep this plan


# The folded tail (tests/test_gpu_fir_fold.py), each case run folded and unfolded.  name: (taps, channels, block, envs,
# plan fields)
FOLD_CASES = {
    "headline_B4096_P32": (131072, 8, F4, {}, dict(P=32, t_batch=4, t_far=0, stagger=1)),
    "B2048_P11": (10 * F2 + 1, 4, F2, {}, dict(P=11, t_batch=4, t_far=0, stagger=0)),
    "B2048_P22": (21 * F2 + 1, 4, F2, {}, dict(P=22, t_batch=4, t_far=0, stagger=1)),
    "B2048_P48": (47 * F2 + 1, 4, F2, {}, dict(P=48, t_batch=4, t_far=8, stagger=0)),
    "B2048_P19_T8": (18 * F2 + 1, 4, F2, dict(DSP_B200_FIR_T=8), dict(P=19, t_batch=8, t_far=0, stagger=0)),
}

# The mid-window pass (tests/test_gpu_fir_pass.py) at the full-wave channel count, each case also run with
# DSP_B200_FIR_PASS=0.  name: (taps, block, P, envs, T, m: DSP_B200_FIR_PASS or None for the default T / 2)
PASS_CASES = {
    "headline_T8_m2": (131072, F4, 32, {}, 8, 2),
    "headline_T8_m4": (131072, F4, 32, {}, 8, None),
    "headline_T8_m6": (131072, F4, 32, {}, 8, 6),
    "headline_T12_m6": (131072, F4, 32, dict(DSP_B200_FIR_T=12), 12, None),
    "B2048_P26": (25 * F2 + 1, F2, 26, {}, 8, None),
    "B2048_P64": (131072, F2, 64, {}, 8, None),
}


# ------------------------------------------------------------------------------------------------------------
# Non-finite samples (tests/test_gpu_nonfinite.py): which output frames may depend on one input frame n
# ------------------------------------------------------------------------------------------------------------
def fir_b0(hint):
    """Level 0's B for calls (or a block hint) of `hint` frames: fir_schedule() (fir_plan.h)."""
    B = 64
    while 2 * B <= hint and B < 8192:
        B *= 2
    return B


def fir_level_taps(levels, taps):
    """[(B, tap0, tap1)] per level of a describe() plan: level 0 from tap 0, level l > 0 from tap B_l, every level
    P_l partitions of B_l taps, the last one ending at the filter's end (fir_schedule())."""
    out = []
    for i, L in enumerate(levels):
        t0 = 0 if i == 0 else L["B"]
        out.append((L["B"], t0, min(taps, t0 + L["P"] * L["B"])))
    return out


def fir_nan_window(n, taps, levels, latency=0):
    """[first, end): the output frames of one FIR channel that may differ when its input frame n changes.
    A level of block B sums, for output block m (frames m B .. m B + B - 1, before the latency), X_{m - tap0/B - p} H_p
    over its partitions p < P, where X_j is the 2B-point transform of input blocks j - 1 and j.  An FFT spreads a
    non-finite input over every bin, so X_k and X_{k+1} (k = n // B) are wholly non-finite, and so is every output block
    they reach:
      - first: level 0 (tap0 = 0) reaches output block n // B0 from its start; an upper level starts at tap0 = B
        and reaches block k + 2 at the earliest, after n.  So first = B0 floor(n / B0) + latency, and nothing earlier
        may differ (the head kernel of a ragged call, a time-domain product, is later than that too).
      - end: the last level (B = B_last, P partitions from tap0) reaches up to output block k + 1 + tap0/B + P - 1,
        which ends at (k + 1) B + tap0 + P B <= (k + 2) B + taps - 1 <= n + 2 B + taps - 1; lower levels end earlier.
        So end = n + taps + 2 B_last + latency, with a margin of (n mod B_last) + (tap0 + P B_last - taps) + 1.
    Every tier, look-ahead and pass of the schedule (fir_plan.h) only re-associates those sums, so stale state that
    the schedule reads with a zero weight is what would break these bounds."""
    B0, Bl = levels[0]["B"], levels[-1]["B"]
    return n // B0 * B0 + latency, n + taps + 2 * Bl + latency


def rs_expect_launch(C, force, oframes, sms):
    """The launch of a resampler call that emits `oframes` frames on C channels, with DSP_B200_RS_TILE=`force` (0:
    unset), on a device of `sms` SMs -- rs_launch() of dsp_b200/csrc/resample_plan.h, restated.  Tiles 1..3 are the FMA
    kernel's R x CH register tiles on a fixed number of warps; 4 is the tensor-core kernel, 5..7 its double-buffered
    form (7 is the default wherever C % 4 == 0, else 2 on even C, else 3; a forced tile the channel count cannot use
    falls back to it).  The tensor-core kernels take 4 warps (128 channels) per CTA while that still leaves 3 CTAs per SM,
    else 2 warps while that leaves 2, else 1.  depth: input-row steps requested ahead (0 on the FMA kernel); minb: CTAs
    per SM of the instantiation's launch bounds; Q: output frames per CTA; channels: channels per CTA."""
    usable = {1: C % 4 == 0, 2: C % 2 == 0, 3: True, 4: C % 4 == 0, 5: C % 4 == 0, 6: C % 4 == 0, 7: C % 4 == 0}
    tile = force if usable.get(force, False) else 7 if C % 4 == 0 else 2 if C % 2 == 0 else 3
    fma = {1: (16, 4, 4, 2), 2: (16, 2, 2, 6), 3: (8, 1, 4, 4)}   # R, CH, warps, minb of k_rs_poly
    if tile in fma:
        R, CH, warps, minb = fma[tile]
        return dict(tile=tile, kernel="k_rs_poly", warps=warps, depth=0, minb=minb, Q=R * warps, channels=32 * CH)
    ctas = lambda w: -(-oframes // 32) * -(-C // (32 * w))
    warps = 4 if C >= 128 and ctas(4) >= 3 * sms else 2 if C >= 64 and ctas(2) >= 2 * sms else 1
    if tile == 4:
        kernel, depth, minb = "k_rs_mma", 1, 4 if warps == 4 else 1
    else:
        kernel, depth = "k_rs_mma2", 3 if tile == 6 and warps == 4 else 2
        minb = {5: 4, 6: 3, 7: 3}[tile] if warps == 4 else 1
    return dict(tile=tile, kernel=kernel, warps=warps, depth=depth, minb=minb, Q=32, channels=32 * warps)


def rs_nan_windows(n, counts, n_, d, in_len, out_delay, Q):
    """(exact, tile): boolean masks over the emitted outputs (calls of `counts` frames, drain polls included) of which
    outputs read input frame n.  exact: n in the output's own window floor(m d / n_) - in_len + 1 .. floor(m d / n_),
    m = out_delay + q (resample.cu header).  tile: n in the rows the output's CTA tile reads.  A launch covers one
    call's outputs in tiles of Q, the first at the call's first output; each tile walks the input rows down from the
    window end of its last output, i_top, to the window start of its first, i_bot (not below row 0), in steps of 4 rows
    (k_rs_poly's RS_G-row stages, the DMMA's k = 4), and multiplies every row with every output's tap -- zero where
    the row is outside that output's window (G's rows are zero-padded) or past i_bot.  0 x NaN = NaN, so a non-finite
    input reaches every output of the tiles that read it: up to Q - 1 outputs before its exact window, and outputs
    up to 3 rows past it."""
    q = np.arange(int(np.sum(counts)), dtype=np.int64)
    ih = (out_delay + q) * d // n_
    exact = (ih - in_len + 1 <= n) & (n <= ih)
    tile = np.zeros(q.size, dtype=bool)
    pos = 0
    for k in counts:
        for a in range(pos, pos + k, Q):
            b = min(a + Q, pos + k) - 1
            top, bot = ih[b], max(ih[a] - in_len + 1, 0)
            if top - 4 * -(-(top - bot + 1) // 4) + 1 <= n <= top:
                tile[a:b + 1] = True
        pos += k
    return exact, tile
